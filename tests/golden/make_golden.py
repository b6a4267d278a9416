"""Generates the committed golden fixtures by running the REFERENCE's own code in the authoring
container (where the reference checkout exists, oracle/build_ref.REF).  Re-run: python tests/golden/make_golden.py

  nms_golden.npz     keep lists of the reference CPU extension (nms_rotated_cpu.cpp, `>=`, host hull) built
                     from the reference checkout into oracle/_ref, on seeded inputs; each case is margin-checked
                     (no decisive IoU within 1e-4 of thr) so the `>`/`>=` and FMA differences cannot flip it
  iou_golden.npz     single_box_iou_rotated<float> host values (through a 2-box NMS probe is not possible,
                     so values come from the pinned C++ oracle, which the pin test ties to the reference
                     extension keep-for-keep) plus the SURVEY §8(c) known-answer case
"""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
import oracle  # noqa: E402
from oracle.build_ref import build, load_ref  # noqa: E402
from tests.boxgen import rboxes, degenerate_pairs  # noqa: E402

OUT = Path(__file__).resolve().parent


def margin_ok(d, s, thr, keep):
    A = np.repeat(d[keep], len(d), 0)
    B = np.tile(d, (len(keep), 1))
    v0 = oracle.iou_pairs(A, B, 0)
    v1 = oracle.iou_pairs(A, B, 1)
    return not (np.any(np.abs(v0 - thr) < 1e-4) or np.any(np.abs(v1 - thr) < 1e-4))


def main():
    assert build(), "needs the reference checkout (oracle/build_ref.REF)"
    ref = load_ref()
    out = {}
    cases = [("dense300", 300, 200, 0.4, 2), ("dense1000", 1000, 300, 0.45, 3), ("cls15_2000", 2000, 1024, 0.4, 15),
             ("lowthr", 800, 300, 0.1, 2), ("highthr", 800, 150, 0.7, 1), ("blockedge", 129, 120, 0.3, 1)]
    for name, n, span, thr, ncls in cases:
        seed = 100
        while True:
            d, s, _ = rboxes(n, span, seed, n_classes=ncls)
            keep = ref.nms_rotated_cpu(torch.from_numpy(d), torch.from_numpy(s), thr).numpy()
            if margin_ok(d, s, thr, keep):
                break
            seed += 1
        assert np.array_equal(keep, oracle.nms_rotated(d, s, thr, 0))
        assert np.array_equal(keep, oracle.nms_rotated(d, s, thr, 1))
        out[f"{name}/dets"], out[f"{name}/scores"] = d, s
        out[f"{name}/thr"], out[f"{name}/keep_cpu"] = np.float32(thr), keep
        print(name, "seed", seed, "n", n, "kept", len(keep))
    # SURVEY §8(c) KAT
    import math
    d = np.array([[136.6, 111.6, 200, 100, -60 * math.pi / 180], [136.6, 111.6, 100, 200, -30 * math.pi / 180],
                  [100, 100, 141.4, 141.4, -45 * math.pi / 180], [100, 100, 141.4, 141.4, 45 * math.pi / 180],
                  [300, 300, 50, 20, 0.3]], np.float32)
    s = np.array([.9, .8, .7, .6, .5], np.float32)
    for thr in (0.1, 0.4, 0.9):
        keep = ref.nms_rotated_cpu(torch.from_numpy(d), torch.from_numpy(s), thr).numpy()
        nm = f"kat{int(thr * 10)}"
        out[f"{nm}/dets"], out[f"{nm}/scores"], out[f"{nm}/thr"], out[f"{nm}/keep_cpu"] = d, s, np.float32(thr), keep
        print(nm, keep)
    np.savez_compressed(OUT / "nms_golden.npz", **out)

    a, b = degenerate_pairs()
    d1, _, _ = rboxes(300, 200, 5, class_offset=False)
    d2, _, _ = rboxes(300, 200, 6, class_offset=False)
    a, b = np.concatenate([a, d1]), np.concatenate([b, d2])
    np.savez_compressed(OUT / "iou_golden.npz", a=a, b=b, iou_host=oracle.iou_pairs(a, b, 0),
                        iou_devorder=oracle.iou_pairs(a, b, 1))


if __name__ == "__main__":
    main()
