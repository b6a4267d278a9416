"""Builds liby5obb.so (all CUDA kernels + the C ABI) for sm_90a (H100) with nvcc, in-tree.

nvcc cross-compiles without a GPU; the .so and the objects are build products (git-ignored).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
OBJ = PKG.parent / "build" / "obj"
LIB = PKG / "liby5obb.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]


def _newer(a: Path, b: Path) -> bool:
    return (not b.exists()) or a.stat().st_mtime > b.stat().st_mtime


def build_lib(force: bool = False, verbose: bool = False) -> Path:
    srcs = sorted(CSRC.glob("*.cu"))
    hdrs = list(CSRC.glob("*.cuh")) + list((PKG.parent / "include").glob("*.h"))
    hdr_m = max(h.stat().st_mtime for h in hdrs)
    OBJ.mkdir(parents=True, exist_ok=True)
    jobs = []
    for s in srcs:
        o = OBJ / (s.stem + ".o")
        if force or _newer(s, o) or o.stat().st_mtime < hdr_m:
            jobs.append((s, o))

    def cc(job):
        s, o = job
        cmd = ["nvcc", *NVCC_FLAGS, "-c", str(s), "-o", str(o)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {s.name}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr, file=sys.stderr)

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            list(ex.map(cc, jobs))
    objs = [OBJ / (s.stem + ".o") for s in srcs]
    if jobs or not LIB.exists():
        cmd = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", str(LIB), *map(str, objs)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build_lib(force="--force" in sys.argv, verbose="-v" in sys.argv))
