"""Golden vectors for DOTA Task1 evaluation (yolov5_obb_b200/dota_eval.py), produced by the REFERENCE's own
DOTA_devkit/dota_evaluation_task1.py voc_eval and voc_ap, with its `polyiou` module backed by the reference's polyiou.cpp
(oracle/_ref/libref_polyiou.so) and matplotlib stubbed by ref_import.

Inputs, written as files and stored as text: labelTxt files for dataset/dataset_demo/labelTxt/P0032.txt (the data fixture
eval_labels_P0032.txt) and five synthetic images with the imagesource: / gsd: header lines, difficult flags 0 / 1 / 2, a class
outside classnames and a duplicated object; Task1 files with unique full-precision scores (so that the reference's order is
defined) for detections jittered from the GTs plus false positives, including a class with no GT (roundabout), a class whose
file is empty (harbor) and a class without a file (helicopter).

Recorded per metric (VOC07, continuous) and ovthresh (0.5, 0.7): rec, prec and ap per class and main()'s mAP.  voc_eval
itself stops with an IndexError on an empty Task1 file (np.array of no rows is 1-D); that class is recorded with an empty
curve and voc_ap of it (0.0 under both metrics), and counts in the mAP as a class whose file exists.
python tests/golden/make_eval_golden.py"""
import contextlib
import io
import sys
import tempfile
import types
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import ref_import  # noqa: E402

CLASSNAMES = ["plane", "ship", "small-vehicle", "large-vehicle", "harbor", "helicopter", "roundabout"]
SYNTH = ["S0001", "S0002", "S0003", "S0004", "S0005"]
METRICS = [(True, 0.5), (False, 0.5), (True, 0.7), (False, 0.7)]


def _rect(rng, W, H):
    cx, cy = rng.uniform(40, W - 40), rng.uniform(40, H - 40)
    l, s = rng.uniform(10, 80), rng.uniform(6, 40)
    th = rng.uniform(-np.pi / 2, np.pi / 2) if rng.random() < 0.6 else 0.0
    c, si = np.cos(th), np.sin(th)
    pts = [(cx + dx * c - dy * si, cy + dx * si + dy * c) for dx, dy in ((-l, -s), (l, -s), (l, s), (-l, s))]
    return np.round(np.array(pts).reshape(-1), 1)


def _fmt(v):
    return " ".join(str(float(x)) for x in v)


def synth_labels(rng):
    out = {}
    for k, name in enumerate(SYNTH):
        lines = ["imagesource:GoogleEarth", "gsd:0.146343590398"]
        for _ in range(int(rng.integers(6, 14))):
            cls = ["plane", "ship", "small-vehicle", "large-vehicle", "harbor", "helicopter", "bridge"][int(rng.integers(0, 7))]
            diff = int(rng.choice([0, 0, 0, 0, 1, 2]))
            lines.append(f"{_fmt(_rect(rng, 1000, 800))} {cls} {diff}")
        if k == 1:
            lines.append(lines[-1])   # a duplicated object: tied IoUs, the first GT wins
        out[name] = "\n".join(lines) + "\n"
    return out


def jitter(rng, poly, s):
    p = np.asarray(poly, np.float64).reshape(4, 2)
    c = p.mean(0)
    p = (p - c) * rng.uniform(0.85, 1.15) + c + rng.normal(0, s, 2)
    return np.round(p.reshape(-1) + rng.normal(0, s / 4, 8), 1)


def synth_dets(rng, labels):
    per_class = {c: [] for c in CLASSNAMES}
    for img, text in labels.items():
        for line in text.splitlines():
            tok = line.split(" ")
            if len(tok) < 9 or tok[8] not in ("plane", "ship", "small-vehicle", "large-vehicle"):
                continue
            for _ in range(int(rng.choice([0, 1, 1, 2, 3]))):
                per_class[tok[8]].append((img, jitter(rng, [float(t) for t in tok[:8]], float(rng.choice([0.5, 2.0, 5.0])))))
    names = list(labels)
    for cls in ("plane", "ship", "small-vehicle", "large-vehicle", "roundabout"):
        for _ in range(int(rng.integers(4, 12))):
            per_class[cls].append((names[int(rng.integers(0, len(names)))], _rect(rng, 1000, 800)))
    out = {}
    for cls, dets in per_class.items():
        if cls == "helicopter":
            continue   # no file
        order = rng.permutation(len(dets))
        out[cls] = "".join(f"{dets[i][0]} {float(rng.uniform(0.01, 1.0))!r} {_fmt(dets[i][1])}\n" for i in order)
    return out


def main():
    ref_import.setup()
    from oracle.build_ref import REF, build_polyiou, load_polyiou
    assert build_polyiou()
    lib = load_polyiou()

    def iou_poly(a, b):
        o = np.zeros(1)
        a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
        lib.ref_iou_poly_pairs(a.ctypes.data, b.ctypes.data, o.ctypes.data, 1)
        return o[0]

    polyiou = types.ModuleType("polyiou")
    polyiou.VectorDouble = list
    polyiou.iou_poly = iou_poly
    sys.modules["polyiou"] = polyiou
    sys.path.insert(0, str(REF / "DOTA_devkit"))
    import dota_evaluation_task1 as DE

    rng = np.random.default_rng(7)
    labels = {"P0032": (HERE / "eval_labels_P0032.txt").read_text()}
    labels.update(synth_labels(rng))
    task1 = synth_dets(rng, labels)
    task1["harbor"] = ""
    imagenames = list(labels)
    work = Path(tempfile.mkdtemp(prefix="eval_golden_"))
    (work / "labelTxt").mkdir()
    for name, text in labels.items():
        (work / "labelTxt" / f"{name}.txt").write_text(text)
    for cls, text in task1.items():
        (work / f"Task1_{cls}.txt").write_text(text)
    (work / "imgnamefile.txt").write_text("\n".join(imagenames) + "\n")
    annopath, detpath, imageset = str(work / "labelTxt" / "{:s}.txt"), str(work / "Task1_{:s}.txt"), str(work / "imgnamefile.txt")

    out = {"imagenames": np.array(imagenames), "classnames": np.array(CLASSNAMES),
           "present": np.array([c in task1 for c in CLASSNAMES])}
    out.update({f"labels/{k}": np.array(v) for k, v in labels.items()})
    out.update({f"task1/{k}": np.array(v) for k, v in task1.items()})
    # the reference's parse of the ground truth (parse_gt), restricted to classnames
    gt_img, gt = [], []
    for i, name in enumerate(imagenames):
        for obj in DE.parse_gt(annopath.format(name)):
            if obj["name"] in CLASSNAMES:
                gt_img.append(i)
                gt.append([float(CLASSNAMES.index(obj["name"])), float(obj["difficult"])] + obj["bbox"])
    out["parse/gt_img"], out["parse/gt"] = np.array(gt_img, np.int32), np.array(gt, np.float64)
    # the Task1 lines as voc_eval splits and converts them (:147-154), classes in order
    det_img, det = [], []
    for c, cls in enumerate(CLASSNAMES):
        for x in task1.get(cls, "").splitlines(keepends=True):
            x = x.strip().split(" ")
            det_img.append(imagenames.index(x[0]))
            det.append([float(c), float(x[1])] + [float(z) for z in x[2:]])
    out["parse/det_img"], out["parse/det"] = np.array(det_img, np.int32), np.array(det, np.float64).reshape(-1, 10)

    for use07, thr in METRICS:
        key = f"eval/{'voc07' if use07 else 'cont'}/{thr}"
        aps, m, skipped = [], 0, 0
        for c, cls in enumerate(CLASSNAMES):
            if cls not in task1:   # main(): a missing file is skipped
                skipped += 1
                aps.append(np.nan)
                continue
            try:
                with contextlib.redirect_stdout(io.StringIO()):
                    rec, prec, ap = DE.voc_eval(detpath, annopath, imageset, cls, ovthresh=thr, use_07_metric=use07)
            except IndexError:
                assert task1[cls] == ""
                rec, prec = np.zeros(0), np.zeros(0)
                ap = DE.voc_ap(rec, prec, use07)
            out[f"{key}/rec/{c}"], out[f"{key}/prec/{c}"] = np.asarray(rec, np.float64), np.asarray(prec, np.float64)
            aps.append(float(ap))
            m = m + ap
        out[f"{key}/ap"] = np.array(aps, np.float64)
        out[f"{key}/map"] = np.float64(m / (len(CLASSNAMES) - skipped))
    np.savez_compressed(HERE / "eval_golden.npz", **out)
    print({k: v.tolist() for k, v in out.items() if k.endswith("/ap") or k.endswith("/map")})
    print("detections", len(det), "gts", len(gt))


if __name__ == "__main__":
    main()
