"""Training-augmentation timing (dev tool): B = 16, S = 1024, hyp.finetune_dota.yaml's probabilities (mosaic 0.75,
mixup 0.1), a synthetic cached set of 1024^2 images with up to 60 labels each.  Reports as one JSON line:
  device_ms_per_batch   CUDA-event time of the two augmentation launches + scan per batch (plans drawn beforehand)
  plan_ms_per_batch     host time of the per-sample Python plan (the random draws and matrices) per batch
  loader_ms_per_batch   wall time per batch of DeviceAugmentLoader alone (plan + launches + the nt read)
  ref_cpu_ms_per_batch  the reference's __getitem__ + collate_fn per batch on this host's CPU, when its checkout is
                        importable here (tests/golden/ref_import.py); null otherwise (not measured)
and the card's name and power limit, read in the same run.
python tools/time_augment.py [batches]"""
import json
import random
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from tests.augmentgen import HYP_DOTA, synth_dataset  # noqa: E402
from yolov5_obb_b200 import augment as P  # noqa: E402

B, S, N_IMAGES = 16, 1024, 48


def ref_cpu_ms(images, labels, batches):
    try:
        sys.path.insert(0, str(ROOT / "tests" / "golden"))
        import ref_import
        ref_import.setup()
        import utils.datasets as D
        from make_augment_golden import Stand
    except Exception:
        return None
    import make_augment_golden
    make_augment_golden.S = S
    ds = Stand(images, labels, dict(HYP_DOTA))
    ds.img_size, ds.mosaic_border = S, [-S // 2, -S // 2]
    t = time.perf_counter()
    for k in range(batches):
        D.LoadImagesAndLabels.collate_fn([ds[(k * B + i) % N_IMAGES] for i in range(B)])
    return (time.perf_counter() - t) / batches * 1e3


def main():
    nb = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    images, labels = synth_dataset(N_IMAGES, S, 0, max_labels=60)
    dev = torch.device("cuda:0")
    ds = P.DeviceDataset(images, labels, S, dev)
    hyp = dict(HYP_DOTA)
    random.seed(0)
    np.random.seed(0)
    t = time.perf_counter()
    plans = [P.plan_batch(ds, [(k * B + i) % N_IMAGES for i in range(B)], hyp) for k in range(nb)]
    plan_ms = (time.perf_counter() - t) / nb * 1e3
    stage = P._Staging()
    for recs in plans[:3]:                                  # warm-up
        P.launch_batch(ds, recs, stage=stage)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for recs in plans:
        P.launch_batch(ds, recs, stage=stage)
    e1.record()
    torch.cuda.synchronize()
    dev_ms = e0.elapsed_time(e1) / nb
    loader = P.DeviceAugmentLoader(ds, hyp, batch_size=B, seed=0)
    it = iter(loader)
    next(it)
    torch.cuda.synchronize()
    t = time.perf_counter()
    n = 0
    for _ in range(min(nb, len(loader) - 1)):
        next(it)
        n += 1
    torch.cuda.synchronize()
    loader_ms = (time.perf_counter() - t) / max(n, 1) * 1e3
    out_bytes = B * 3 * S * S
    print(json.dumps({"card": card, "B": B, "S": S, "batches": nb, "device_ms_per_batch": round(dev_ms, 3),
                      "plan_ms_per_batch": round(plan_ms, 3), "loader_ms_per_batch": round(loader_ms, 3),
                      "output_GBps": round(out_bytes / dev_ms / 1e6, 1),
                      "ref_cpu_ms_per_batch": (lambda v: None if v is None else round(v, 1))(
                          ref_cpu_ms(images, labels, 2))}))


if __name__ == "__main__":
    main()
