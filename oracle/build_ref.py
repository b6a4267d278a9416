"""Build the reference's own native code for the hot path into oracle/_ref/ (TEST INFRASTRUCTURE ONLY).

Nothing here is product code.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs may load what this script produces.

What gets built, straight from the sources where they lie in the reference checkout (never copied) - the directory named
by $YOLOV5_OBB_REF, by default `reference` next to this repository:

  oracle/_ref/nms_rotated_ref*.so   torch extension = utils/nms_rotated/src/{nms_rotated_cpu.cpp,
                                    nms_rotated_cuda.cu, box_iou_rotated_utils.h} + a 20-line pybind shim
                                    written here (the reference's own nms_rotated_ext.cpp also wants
                                    poly_nms_cuda.cu, which needs THC and cannot build on torch>=1.11).
                                    Exposes nms_rotated_cpu / nms_rotated_cuda exactly as the reference
                                    declares them (src/nms_rotated_ext.cpp:8-22).
  oracle/_ref/libref_iou.so         torch-free nvcc build of a 10-line kernel that instantiates the
                                    reference's single_box_iou_rotated<float> device function
                                    (src/box_iou_rotated_utils.h:334-360) on N pairs, so the GPU tests can
                                    compare IoU values with the reference's.

Without the reference checkout nothing is rebuilt and the files already in oracle/_ref (git-ignored) are used as they are;
the tests that need them skip when they are missing.
"""
import os
import shutil
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
OUT = HERE / "_ref"
REF = Path(os.environ.get("YOLOV5_OBB_REF", HERE.parents[1] / "reference"))
SRC = REF / "utils" / "nms_rotated" / "src"

SHIM = r'''
// pybind shim for the reference kernels (declarations as in utils/nms_rotated/src/nms_rotated_ext.cpp:8-22)
#include <ATen/ATen.h>
#include <torch/extension.h>
at::Tensor nms_rotated_cuda(const at::Tensor& dets, const at::Tensor& scores, const float iou_threshold);
at::Tensor nms_rotated_cpu(const at::Tensor& dets, const at::Tensor& scores, const float iou_threshold);
PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("nms_rotated_cpu", [](const at::Tensor& d, const at::Tensor& s, double t) {
    return nms_rotated_cpu(d.contiguous(), s.contiguous(), (float)t); });
  m.def("nms_rotated_cuda", [](const at::Tensor& d, const at::Tensor& s, double t) {
    return nms_rotated_cuda(d.contiguous(), s.contiguous(), (float)t); });
}
'''

IOU_HARNESS = r'''
// instantiates the reference device function on N independent pairs (test infrastructure)
#include "%(hdr)s"
#include <cuda_runtime.h>
__global__ void ref_iou_pairs_kernel(const float* a, const float* b, float* out, long n) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = single_box_iou_rotated<float>(a + 5 * i, b + 5 * i);
}
extern "C" int ref_iou_pairs(const float* a, const float* b, float* out, long n, void* stream) {
  if (n <= 0) return 0;
  ref_iou_pairs_kernel<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a, b, out, n);
  return (int)cudaGetLastError();
}
'''


def build(force: bool = False) -> bool:
    """Returns True if oracle/_ref is usable afterwards."""
    have = list(OUT.glob("nms_rotated_ref*.so")) and (OUT / "libref_iou.so").exists()
    if not REF.exists():
        return bool(have)
    if have and not force:
        return True
    OUT.mkdir(exist_ok=True)
    work = OUT / "_build"
    work.mkdir(exist_ok=True)
    (work / "ref_shim.cpp").write_text(SHIM)
    (work / "ref_iou_harness.cu").write_text(IOU_HARNESS % {"hdr": str(SRC / "box_iou_rotated_utils.h")})

    # 1) torch-free IoU harness (nvcc defaults, as the reference's own build: FMA contraction on)
    subprocess.check_call([
        "nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-shared", "-Xcompiler", "-fPIC",
        "-o", str(OUT / "libref_iou.so"), str(work / "ref_iou_harness.cu")])

    # 2) the reference torch extension (CPU kernel + CUDA kernel K1), same nvcc defines as the
    #    reference's setup.py:18-22
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "4")
    from torch.utils.cpp_extension import load
    mod = load(
        name="nms_rotated_ref",
        sources=[str(work / "ref_shim.cpp"), str(SRC / "nms_rotated_cpu.cpp"), str(SRC / "nms_rotated_cuda.cu")],
        extra_include_paths=[str(SRC)],
        extra_cuda_cflags=["-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__",
                           "-D__CUDA_NO_HALF2_OPERATORS__"],
        with_cuda=True,
        build_directory=str(work),
        verbose=False,
    )
    so = Path(mod.__file__)
    shutil.copy2(so, OUT / so.name)
    return True


POLY_SHIM = r'''
// C shim around the reference's DOTA_devkit/polyiou.cpp (declared in polyiou.h:9): test infrastructure
#include <vector>
double iou_poly(std::vector<double> p, std::vector<double> q);
extern "C" void ref_iou_poly_pairs(const double* p8, const double* q8, double* out, long n) {
  for (long i = 0; i < n; ++i)
    out[i] = iou_poly(std::vector<double>(p8 + 8 * i, p8 + 8 * i + 8), std::vector<double>(q8 + 8 * i, q8 + 8 * i + 8));
}
'''


def build_polyiou(force: bool = False) -> bool:
    """oracle/_ref/libref_polyiou.so = the reference's DOTA_devkit/polyiou.cpp (the polygon IoU behind the tile-merge NMS,
    ResultMerge_multi_process.py:62-123) compiled in place with g++ plus the C shim above."""
    so = OUT / "libref_polyiou.so"
    if not REF.exists():
        return so.exists()
    if so.exists() and not force:
        return True
    OUT.mkdir(exist_ok=True)
    work = OUT / "_build"
    work.mkdir(exist_ok=True)
    (work / "ref_polyiou_shim.cpp").write_text(POLY_SHIM)
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-ffp-contract=off", "-o", str(so),
                           str(work / "ref_polyiou_shim.cpp"), str(REF / "DOTA_devkit" / "polyiou.cpp")])
    return True


POLYGPU_SHIM = r'''
// extern "C" doors to the reference's C++ entry points (poly_nms.hpp:9-10, poly_overlaps.hpp:1): test infrastructure
void %(decl)s;
extern "C" void ref_%(name)s(%(params)s) { %(call)s; }
'''


def build_polygpu(force: bool = False) -> bool:
    """oracle/_ref/libref_polygpu_{nms,overlaps}.so = the reference's DOTA_devkit/poly_nms_gpu/poly_nms_kernel.cu and
    poly_overlaps_kernel.cu compiled unmodified, in place, for sm_90a (the reference's setup.py passes -arch=sm_35 and no
    other code-generation flag).  Two libraries: both files define `_set_device`."""
    outs = {"nms": OUT / "libref_polygpu_nms.so", "overlaps": OUT / "libref_polygpu_overlaps.so"}
    if not REF.exists():
        return all(o.exists() for o in outs.values())
    if all(o.exists() for o in outs.values()) and not force:
        return True
    OUT.mkdir(exist_ok=True)
    work = OUT / "_build"
    work.mkdir(exist_ok=True)
    src = REF / "DOTA_devkit" / "poly_nms_gpu"
    spec = {
        "nms": ("poly_nms_kernel.cu",
                dict(decl="_poly_nms(int*, int*, const float*, int, int, float, int)", name="poly_nms",
                     params="int* keep, int* num, const float* polys, int n, int dim, float thr, int dev",
                     call="_poly_nms(keep, num, polys, n, dim, thr, dev)")),
        "overlaps": ("poly_overlaps_kernel.cu",
                     dict(decl="_overlaps(float*, const float*, const float*, int, int, int)", name="overlaps",
                          params="float* ov, const float* b, const float* q, int n, int k, int dev",
                          call="_overlaps(ov, b, q, n, k, dev)")),
    }
    for key, (cu, d) in spec.items():
        shim = work / f"ref_polygpu_{key}_shim.cpp"
        shim.write_text(POLYGPU_SHIM % d)
        subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC", "-w",
                               "-I", str(src), "-o", str(outs[key]), str(src / cu), str(shim)])
    return True


def load_polygpu():
    import ctypes
    libs = {}
    for key in ("nms", "overlaps"):
        so = OUT / f"libref_polygpu_{key}.so"
        if not so.exists():
            raise FileNotFoundError(f"{so} not built; run python oracle/build_ref.py")
        libs[key] = ctypes.CDLL(str(so))
    vp, ci, cf = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    libs["nms"].ref_poly_nms.argtypes = [vp, vp, vp, ci, ci, cf, ci]
    libs["nms"].ref_poly_nms.restype = None
    libs["overlaps"].ref_overlaps.argtypes = [vp, vp, vp, ci, ci, ci]
    libs["overlaps"].ref_overlaps.restype = None
    return libs["nms"].ref_poly_nms, libs["overlaps"].ref_overlaps


def load_polyiou():
    import ctypes
    so = OUT / "libref_polyiou.so"
    if not so.exists():
        raise FileNotFoundError("oracle/_ref/libref_polyiou.so not built; run python oracle/build_ref.py")
    lib = ctypes.CDLL(str(so))
    lib.ref_iou_poly_pairs.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_long]
    lib.ref_iou_poly_pairs.restype = None
    return lib


def load_ref():
    """Import the prebuilt reference extension (tests only)."""
    import importlib.util
    import torch  # noqa: F401  (the extension links against libtorch)
    sos = sorted(OUT.glob("nms_rotated_ref*.so"))
    if not sos:
        raise FileNotFoundError("oracle/_ref/nms_rotated_ref*.so not built; run python oracle/build_ref.py")
    spec = importlib.util.spec_from_file_location("nms_rotated_ref", sos[0])
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    ok = build(force="--force" in sys.argv)
    ok2 = build_polyiou(force="--force" in sys.argv)
    ok3 = build_polygpu(force="--force" in sys.argv)
    print("oracle/_ref:", "ok" if ok else "unavailable", "| polyiou:", "ok" if ok2 else "unavailable",
          "| devkit poly_nms_gpu:", "ok" if ok3 else "unavailable")
