"""DOTA Task1 evaluation timing (dev tool): a DOTA-val-sized synthetic set, 458 scenes of 2000 x 2000 with 15 classes, whose
detections come from the tile merge (merge_tiles over tests/scenegen.tile_rows, 9 tiles per scene) and whose ground truth is
a jittered 70 % of them (10 % difficult) plus missed objects.  Reports the CUDA-event time of evaluate_task1 (VOC07 and
continuous AP, ovthresh 0.5, all classes) and the host time of the CPU restatement oracle/eval_ref.py, which loops over the
detections in Python like the reference's voc_eval, on the first `cpu_scenes` scenes only (labelled as such), with the card's
name and power limit.  python tools/time_eval.py [reps] [cpu_scenes]"""
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import eval_ref  # noqa: E402
from tests.scenegen import tile_rows  # noqa: E402
from yolov5_obb_b200.dota_eval import GroundTruth, Task1Detections, evaluate_task1  # noqa: E402
from yolov5_obb_b200.scene import merge_tiles  # noqa: E402

N_SCENES, NC, SIDE = 458, 15, 2000


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    cpu_scenes = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    names = [f"S{i:04d}" for i in range(N_SCENES)]
    dets = Task1Detections(names, NC, dev)
    rng = np.random.default_rng(0)
    gt_img, gt = [], []
    for i in range(N_SCENES):
        origins, rows, counts = tile_rows(SIDE, SIDE, 600, nc=NC, seed=1000 + i, max_det=1500)
        sc = merge_tiles(torch.from_numpy(rows).to(dev), torch.from_numpy(counts).to(dev), torch.from_numpy(origins).to(dev),
                         NC, 16.0, 0.2)
        dets.add(i, sc)
        r = sc.rows.cpu().numpy()
        keep = r[rng.random(len(r)) < 0.7]
        miss = r[rng.integers(0, len(r), len(r) // 10)].copy()
        miss[:, 2:] += 300.0
        g = np.concatenate([keep, miss])
        g[:, 2:] = np.round(g[:, 2:] + rng.normal(0, 1.5, (len(g), 8)), 1)
        g[:, 1] = (rng.random(len(g)) < 0.1).astype(np.float64)
        gt.append(g)
        gt_img.append(np.full(len(g), i, np.int32))
    gt_img, gt = np.concatenate(gt_img), np.concatenate(gt)
    truth = GroundTruth(torch.from_numpy(gt_img).to(dev), torch.from_numpy(gt).to(dev), names, NC)
    det_img, det_rows = dets.img, dets.rows
    out = {"card": card, "scenes": N_SCENES, "classes": NC, "detections": int(det_rows.shape[0]), "ground_truths": len(gt)}
    for use07 in (True, False):
        for _ in range(2):
            evaluate_task1(dets, truth, 0.5, use07).check()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(reps):
            res = evaluate_task1(dets, truth, 0.5, use07)
        ev[1].record()
        torch.cuda.synchronize()
        out[f"device_ms_{'voc07' if use07 else 'continuous'}"] = round(ev[0].elapsed_time(ev[1]) / reps, 3)
        out[f"map_{'voc07' if use07 else 'continuous'}"] = res.map

    # the CPU restatement on a subset of the scenes, against the device on the same subset
    di, dr = det_img.cpu().numpy(), det_rows.cpu().numpy()
    ds, gs = di < cpu_scenes, gt_img < cpu_scenes
    sub = Task1Detections(names[:cpu_scenes], NC, dev).add_rows(det_img[torch.from_numpy(ds).to(dev)],
                                                                det_rows[torch.from_numpy(ds).to(dev)])
    sub_gt = GroundTruth(truth.img[torch.from_numpy(gs).to(dev)], truth.rows[torch.from_numpy(gs).to(dev)], names[:cpu_scenes], NC)
    t0 = time.perf_counter()
    want = eval_ref.evaluate(di[ds], dr[ds], gt_img[gs], gt[gs], NC, 0.5, True)
    host_s = time.perf_counter() - t0
    got = evaluate_task1(sub, sub_gt, 0.5, True)
    assert np.array_equal(got.ap.cpu().numpy(), want["ap"], equal_nan=True)
    out.update({"cpu_subset_scenes": cpu_scenes, "cpu_subset_detections": int(ds.sum()),
                "cpu_restatement_subset_ms": round(host_s * 1e3, 1)})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
