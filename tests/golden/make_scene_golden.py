"""Golden vectors for whole-scene inference (yolov5_obb_b200/scene.py), produced by the REFERENCE's own code:
  * split origins: DOTA_devkit/ImgSplit_multi_process.py splitbase.SplitSingle at rate 1 with `savepatches` recording
    (left, up) (cv2.imread returns a blank scene of the requested size; no label file);
  * tile merge: per-tile detections -> utils/rboxs_utils.rbox2poly, utils/general.scale_polys (pad 16, 1056^2 tiles) ->
    val.py save_one_json -> json -> tools/TestJson2VocClassTxt.py -> DOTA_devkit/ResultMerge_multi_process.py mergesingle with
    py_cpu_nms_poly_fast over the reference's polyiou.cpp (oracle/_ref/libref_polyiou.so); the NMS input and keep list of
    every class file are recorded, and the Task1 text mergesingle writes.
python tests/golden/make_scene_golden.py"""
import ctypes
import json
import subprocess
import sys
import tempfile
import types
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import ref_import  # noqa: E402

ROOT = HERE.parents[1]
SPLIT_SIZES = [(700, 900), (1024, 1024), (1024, 1025), (1025, 1024), (1848, 2672), (1000, 1848), (4000, 4000),
               (20000, 20000), (1700, 2300), (3000, 800), (824, 1024), (1648, 1649)]
MERGE_SCENE = (1700, 2300)


def stub_shapely():
    sh = types.ModuleType("shapely")
    sh.geometry = types.ModuleType("shapely.geometry")
    sys.modules["shapely"] = sh
    sys.modules["shapely.geometry"] = sh.geometry


def split_golden(REF):
    sys.path.insert(0, str(REF / "DOTA_devkit"))
    import ImgSplit_multi_process as IS
    out = {}
    for H, W in SPLIT_SIZES:
        rec = []
        sb = object.__new__(IS.splitbase)
        sb.subsize, sb.gap = 1024, 200
        sb.slide = sb.subsize - sb.gap
        sb.imagepath = sb.labelpath = "/nonexistent"
        sb.savepatches = lambda img, objs, name, left, up, right, down: rec.append((left, up))
        IS.cv2 = types.SimpleNamespace(imread=lambda p, H=H, W=W: np.broadcast_to(np.zeros(1, np.uint8), (H, W, 3)))
        IS.util.parse_dota_poly2 = lambda f: []
        sb.SplitSingle("P0000", 1, ".png")
        out[f"split/{H}x{W}"] = np.array(rec, np.int64).reshape(-1, 2)
    return out


def merge_golden(REF):
    from oracle.build_ref import build_polyiou, load_polyiou
    from tests.scenegen import tile_rows
    assert build_polyiou()
    lib = load_polyiou()

    def iou_poly(a, b):
        o = np.zeros(1)
        a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
        lib.ref_iou_poly_pairs(a.ctypes.data, b.ctypes.data, o.ctypes.data, 1)
        return o[0]

    polyiou = types.ModuleType("DOTA_devkit.polyiou")
    polyiou.VectorDouble = list
    polyiou.iou_poly = iou_poly
    sys.modules["DOTA_devkit.polyiou"] = polyiou
    from utils.general import scale_polys
    from utils.rboxs_utils import rbox2poly, poly2hbb
    import val
    from DOTA_devkit import ResultMerge_multi_process as RM

    H, W = MERGE_SCENE
    origins, rows, counts = tile_rows(H, W, 420, nc=15, seed=3, rotated=False)
    jdict, polys_all = [], np.zeros(rows.shape[:2] + (8,), np.float32)
    for t, (left, up) in enumerate(origins.tolist()):
        r = torch.from_numpy(rows[t, :counts[t]])
        poly = rbox2poly(r[:, :5])
        poly = scale_polys((1056, 1056), poly, (1024, 1024), ratio_pad=((1.0, 1.0), (16.0, 16.0)))
        polys_all[t, :counts[t]] = poly.numpy()
        hbb = poly2hbb(poly)
        xyxy = torch.cat([hbb[:, :2] - hbb[:, 2:] / 2, hbb[:, :2] + hbb[:, 2:] / 2], 1)
        val.save_one_json(torch.cat([xyxy, r[:, 5:7]], 1), torch.cat([poly, r[:, 5:7]], 1), jdict,
                          Path(f"P0000__1__{left}___{up}.png"), list(range(1000)))
    work = Path(tempfile.mkdtemp(prefix="scene_golden_"))
    (work / "pred.json").write_text(json.dumps(jdict))
    subprocess.check_call([sys.executable, str(REF / "tools" / "TestJson2VocClassTxt.py"), "--json_path",
                           str(work / "pred.json"), "--save_path", str(work / "txt")], cwd=str(work))
    (work / "merged").mkdir()
    out = {"merge/origins": origins, "merge/rows": rows, "merge/counts": counts, "merge/polys": polys_all}
    names = ['plane', 'baseball-diamond', 'bridge', 'ground-track-field', 'small-vehicle', 'large-vehicle', 'ship',
             'tennis-court', 'basketball-court', 'storage-tank', 'soccer-ball-field', 'roundabout', 'harbor', 'swimming-pool',
             'helicopter', 'container-crane']  # TestJson2VocClassTxt.py's DOTA_CLASSES (v1.5)
    merged = []
    for c, name in enumerate(names):
        f = work / "txt" / f"Task1_{name}.txt"
        if not f.exists():
            continue
        seen = []

        def nms(dets, thresh):
            keep = RM.py_cpu_nms_poly_fast(dets, thresh)
            seen.append(dets[keep])
            return keep

        RM.mergesingle(str(work / "merged"), nms, str(f))
        assert len(seen) == 1
        kept = seen[0]
        merged.append(np.concatenate([np.full((len(kept), 1), float(c)), kept[:, 8:9], kept[:, :8]], 1))
        out[f"merge/text/{c}"] = np.array((work / "merged" / f.name).read_text())
    out["merge/merged"] = np.concatenate(merged, 0)
    out["merge/names"] = np.array(names)
    return out


def main():
    ref_import.setup()
    from oracle.build_ref import REF
    stub_shapely()
    out = split_golden(REF)
    out.update(merge_golden(REF))
    np.savez_compressed(HERE / "scene_golden.npz", **out)
    print({k: getattr(v, "shape", v) for k, v in out.items() if not k.startswith("merge/text")})


if __name__ == "__main__":
    main()
