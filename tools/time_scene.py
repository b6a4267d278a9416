"""Whole-scene inference timing (dev tool): a synthetic 4000 x 4000 scene (25 tiles of 1024^2, 1056^2 network input) through
SceneDetector with yolov5s at batch 16, conf 0.01, iou 0.4, max_det 1500 (val.py --task test settings).  Reports scenes/s end to
end (host clock around det() + a device synchronise), the CUDA-event time of each stage (tile input, network, per-tile NMS,
merge), and the host merge of the same detections through the CPU restatement (oracle/scene_ref.py), with the card's name and
power limit.  python tools/time_scene.py [reps]"""
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tests.modelgen import calibrated_bench_model  # noqa: E402
from tests.tilegen import synth_tiles  # noqa: E402
from yolov5_obb_b200 import _lib  # noqa: E402
from yolov5_obb_b200.general import DetectRecords, non_max_suppression_obb  # noqa: E402
from yolov5_obb_b200.scene import SceneDetector, merge_tiles, split_origins  # noqa: E402


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    m = calibrated_bench_model("s").to(dev)
    scene = synth_tiles(1, 4000, 7)[0].permute(1, 2, 0).contiguous().to(dev)
    det = SceneDetector(m, batch_size=16)
    for _ in range(3):
        det.det(scene).rows
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        res = det.det(scene)
        res.rows
    torch.cuda.synchronize()
    e2e = (time.perf_counter() - t0) / reps

    # the same work stage by stage, CUDA events between the stages
    L = _lib.lib()
    origins = split_origins(4000, 4000)
    T, B = len(origins), det.B
    org = torch.tensor(origins, dtype=torch.int32, device=dev)
    rows = torch.empty((T, det.max_det, 7), device=dev)
    counts = torch.empty(T, dtype=torch.int64, device=dev)
    eng = m.records_plan((B, 3, det.size, det.size), dev)
    st = _lib.stream_ptr(dev)
    ms = {"tile input": 0.0, "network": 0.0, "per-tile NMS": 0.0, "merge": 0.0}
    for rep in range(reps + 1):
        acc = {k: 0.0 for k in ms}
        for i in range(0, T, B):
            n = min(B, T - i)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[0].record()
            _lib.check(L.y5obb_scene_tiles_s2d_u8(scene.data_ptr(), 4000, 4000, org[i].data_ptr(), n, 1024, det.size,
                                                  det.border, eng.x_s2d.data_ptr(), 1, st), "tiles")
            ev[1].record()
            rec = DetectRecords(eng.forward_s2d(), eng.nc)
            ev[2].record()
            out, c, _ = non_max_suppression_obb(rec, 0.01, 0.4, multi_label=True, max_det=det.max_det, return_packed="async")
            rows[i:i + n].copy_(out[:n])
            counts[i:i + n].copy_(c[:n])
            ev[3].record()
            torch.cuda.synchronize()
            for k, (a, b) in zip(("tile input", "network", "per-tile NMS"), ((0, 1), (1, 2), (2, 3))):
                acc[k] += ev[a].elapsed_time(ev[b])
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        merged = merge_tiles(rows, counts, org, eng.nc, det.pad_xy, det.merge_thresh)
        e1.record()
        torch.cuda.synchronize()
        acc["merge"] = e0.elapsed_time(e1)
        if rep > 0:   # first pass: warm-up
            for k in ms:
                ms[k] += acc[k] / reps
    assert torch.equal(merged.rows, res.rows)

    from oracle import scene_ref
    from yolov5_obb_b200.rboxs_utils import rbox2poly, scale_polys
    tiles = []
    for t, (left, up) in enumerate(origins):
        r = rows[t, :int(counts[t])]
        poly = scale_polys((det.size, det.size), rbox2poly(r[:, :5]), (1024, 1024), ((1.0, 1.0), (det.pad_xy, det.pad_xy)))
        tiles.append((left, up, poly.cpu().numpy(), r[:, 5].cpu().numpy(), r[:, 6].long().cpu().numpy()))
    t0 = time.perf_counter()
    host = scene_ref.merge(tiles, eng.nc, det.merge_thresh)
    host_s = time.perf_counter() - t0
    assert torch.equal(torch.from_numpy(host), res.rows.cpu())
    print(json.dumps({"card": card, "scene": "4000x4000", "tiles": T, "batch": B, "model": "yolov5s",
                      "tile_detections": int(counts.sum()), "merged": int(res.rows.shape[0]),
                      "scenes_per_s": round(1.0 / e2e, 3), "scene_ms": round(e2e * 1e3, 2),
                      "stage_ms": {k: round(v, 3) for k, v in ms.items()},
                      "host_merge_restatement_ms": round(host_s * 1e3, 1)}))


if __name__ == "__main__":
    main()
