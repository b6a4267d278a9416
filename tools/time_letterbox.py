"""Timing of the image front end (dev tool): y5obb_letterbox_s2d_u8 alone at batch 16 -> 1024^2 for four source sizes (CUDA
events over many launches; bytes read + written computed from the shapes, against the 3.35 TB/s HBM3 figure of the H100 SXM
data sheet: the kernel is HBM-bound), and DetectPipeline images/s from host images to host detections for three arms
alternated in the same run: (a) cv2 letterbox on the host feeding DetectPipeline.__call__ (the path without this kernel),
(b) DetectPipeline.run_images, (c) __call__ on tensors letterboxed beforehand (the ceiling).  yolov5s, batch 16, rect mode.
Prints one JSON line with the card's name and power limit.  python tools/time_letterbox.py [reps] [launches]"""
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tests.letterboxgen import synth_image  # noqa: E402
from tests.modelgen import calibrated_bench_model  # noqa: E402
from yolov5_obb_b200 import _lib, general  # noqa: E402
from yolov5_obb_b200 import letterbox as P  # noqa: E402
from yolov5_obb_b200.pipeline import DetectPipeline  # noqa: E402

B, SIZE = 16, 1024
SOURCES = [(1024, 1024), (800, 1333), (1689, 2425), (4000, 4000)]
HBM_PEAK = 3.35e12


def kernel_bytes(places, Hp, Wp):
    """Bytes the algorithm needs: every source byte the resampler touches once (the whole image) + the bf16 stem input."""
    return sum(p.h0 * p.w0 * 3 for p in places) + len(places) * (Hp // 2) * (Wp // 2) * 32


def time_kernel(h0, w0, launches, dev):
    im = synth_image(h0, w0, 1)
    _, shapes = P.rect_batch_shapes([(w0, h0)] * B, B, SIZE, 32, 0.0)
    Hp, Wp = int(shapes[0][0]), int(shapes[0][1])
    places = [P.place_rect(h0, w0, SIZE, (Hp, Wp)) for _ in range(B)]
    batch = P.pack_batch([im] * B, places, Hp, Wp)
    buf = batch.host[:batch.nbytes].to(dev)
    x = torch.zeros((B, Hp // 2, Wp // 2 + 2, 16), dtype=torch.bfloat16, device=dev)
    for _ in range(5):
        P.letterbox_s2d(buf, batch, x, 1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        P.letterbox_s2d(buf, batch, x, 1)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / launches
    nbytes = kernel_bytes(places, Hp, Wp)
    mode = P.resample_plan(h0, w0, places[0].new_h, places[0].new_w, places[0].interp)[0]
    return {"source": f"{h0}x{w0}", "net": f"{Hp}x{Wp}", "mode": ["copy", "linear", "area_int", "area"][mode],
            "ms": round(ms, 4), "MB": round(nbytes / 1e6, 1), "GBps": round(nbytes / ms / 1e6, 1),
            "share_of_hbm_peak": round(nbytes / (ms * 1e-3) / HBM_PEAK, 3)}


def cv2_letterbox_batch(cv2, ims, img_size, shape):
    """val.py's loader on the host: load_image_label's resize + letterbox + transpose, per image (utils/datasets.py)."""
    out = np.empty((len(ims), 3, shape[0], shape[1]), np.uint8)
    for b, im in enumerate(ims):
        h0, w0 = im.shape[:2]
        (h, w), interp, _ = P.load_image_size(h0, w0, img_size)
        if interp is not None:
            im = cv2.resize(im, (w, h), interpolation=cv2.INTER_AREA if interp == P.AREA else cv2.INTER_LINEAR)
        _, (top, bottom, left, right), _, _ = P.letterbox_geometry((h, w), shape, False, False, False)
        im = cv2.copyMakeBorder(im, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(114, 114, 114))
        out[b] = im.transpose((2, 0, 1))[::-1]
    return out


def time_pipeline(h0, w0, n_batches, reps, model, dev):
    try:
        import cv2
        cv2.setNumThreads(1)   # the reference's loader resizes on one thread per worker
    except ImportError:
        cv2 = None
    ims = [synth_image(h0, w0, 10 + i) for i in range(4)]
    images = [ims[i % 4] for i in range(B * n_batches)]
    _, shapes = P.rect_batch_shapes([(w0, h0)] * B, B, SIZE, 32, 0.0)
    shape = (int(shapes[0][0]), int(shapes[0][1]))
    pipe = DetectPipeline(model, 0.25, 0.45, 1500, multi_label=True, device=dev, slots=2)
    pinned = [torch.empty((B, 3) + shape, dtype=torch.uint8).pin_memory() for _ in range(3)]
    pre = None

    def arm_a():
        def gen():
            for i in range(n_batches):
                t = pinned[i % 3]
                t.numpy()[:] = cv2_letterbox_batch(cv2, images[i * B:(i + 1) * B], SIZE, shape)
                yield t
        return sum(len(d) for d in pipe(gen()))

    def arm_b():
        return sum(1 for _ in pipe.run_images(images, img_size=SIZE, stride=32, auto=False, batch_size=B))

    def arm_c():
        return sum(len(d) for d in pipe(iter(pre)))

    if cv2 is not None:
        pre = [torch.from_numpy(cv2_letterbox_batch(cv2, images[i * B:(i + 1) * B], SIZE, shape)).pin_memory()
               for i in range(n_batches)]
    else:   # the ceiling needs letterboxed tensors of the right shape only
        pre = [torch.randint(0, 256, (B, 3) + shape, dtype=torch.uint8).pin_memory() for _ in range(n_batches)]
    arms = {"b_run_images": arm_b, "c_preletterboxed": arm_c}
    if cv2 is not None:
        arms["a_cv2_host_letterbox"] = arm_a
    for f in arms.values():   # plans, graphs and buffers of every arm
        f()
        f()
    rates = {k: [] for k in arms}
    for _ in range(reps):
        for k, f in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n = f()
            torch.cuda.synchronize()
            rates[k].append(n / (time.perf_counter() - t0))
    out = {"source": f"{h0}x{w0}", "images": len(images)}
    for k, v in rates.items():
        out[k] = {"images_per_s": round(statistics.median(v), 1), "min": round(min(v), 1), "max": round(max(v), 1)}
    if cv2 is None:
        out["a_cv2_host_letterbox"] = "not measured (cv2 is not installed)"
    # every network shape keeps its plans, post-process graphs and their workspaces: drop them before the next source size
    del pipe, pre, pinned
    general._GRAPHS.clear()
    _lib._WS.clear()
    model._engines.clear()
    torch.cuda.empty_cache()
    return out


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    launches = int(sys.argv[2]) if len(sys.argv) > 2 else 200
    if not torch.cuda.is_available():
        raise SystemExit("time_letterbox.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    kern = [time_kernel(h, w, launches, dev) for h, w in SOURCES]
    model = calibrated_bench_model("s").to(dev)
    pipe = [time_pipeline(h, w, 6, reps, model, dev) for h, w in SOURCES]
    print(json.dumps({"card": card, "batch": B, "img_size": SIZE, "model": "yolov5s", "kernel": kern, "pipeline": pipe}))


if __name__ == "__main__":
    main()
