"""Goldens for the image front end (yolov5_obb_b200/letterbox.py, csrc/letterbox.cu) from the REFERENCE's own code:
  * utils/augmentations.letterbox geometry over a grid of shapes x (auto, scaleFill, scaleup) x strides (a recording
    cv2.copyMakeBorder / cv2.resize pair gives new_unpad and the borders), and its bytes on the seeded images;
  * utils/datasets.LoadImages on a folder of the seeded images of tests/letterboxgen.py (PNG, lossless) and on
    dataset/dataset_demo (P0032, 2425 x 1689): the CHW RGB image per file;
  * utils/datasets.LoadImagesAndLabels(rect=True, pad=0.5) on the same folder: order, batch shapes, and per item the image,
    the `shapes` entry and the label polygons in network-input pixels.
Every image is kept as the SHA-256 of its bytes plus its shape, which pins the restatement bit for bit; full bytes are kept
only for the subset the GPU tests feed to the device (letterboxgen.GOLDEN_FULL_DETECT / GOLDEN_FULL_RECT_BATCHES).  python tests/golden/make_letterbox_golden.py"""
import hashlib
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import ref_import  # noqa: E402

ref_import.setup()
sys.path.insert(0, str(HERE.parents[1]))
import cv2  # noqa: E402
import utils.augmentations as AUG  # noqa: E402
import utils.datasets as D  # noqa: E402
from oracle.build_ref import REF  # noqa: E402
from tests import letterboxgen as LG  # noqa: E402

GEOM_SHAPES = [(1689, 2425), (1024, 1024), (2048, 2048), (800, 1333), (4000, 4000), (100, 100), (33, 977), (977, 33), (1, 7),
               (1080, 1920), (1023, 1025), (511, 2047), (3000, 2999)]
GEOM_NEW = [640, 1024, (512, 768), (1056, 1056)]


class ClassNames(list):
    """verify_image_label concatenates the class index with the coordinate strings, which the installed numpy refuses for an
    int next to str: hand it the index as a string (np.array(..., dtype=np.float32) parses it back)."""

    def index(self, name):
        return str(list.index(self, name))


def digest(img):
    return np.array(hashlib.sha256(np.ascontiguousarray(img).tobytes()).hexdigest())


def geometry_golden():
    rows = []
    real_resize, real_border = cv2.resize, cv2.copyMakeBorder
    rec = {}
    AUG.cv2.resize = lambda im, size, interpolation=None: (rec.__setitem__("unpad", size), np.zeros((size[1], size[0], 3), np.uint8))[1]
    AUG.cv2.copyMakeBorder = lambda im, t, b, l, r, *a, **k: (rec.__setitem__("border", (t, b, l, r)), im)[1]
    try:
        for shape in GEOM_SHAPES:
            for new in GEOM_NEW:
                for auto in (True, False):
                    for fill in (True, False):
                        for up in (True, False):
                            for stride in (32, 64):
                                rec.clear()
                                _, ratio, pad = AUG.letterbox(np.zeros(shape + (3,), np.uint8), new, auto=auto, scaleFill=fill,
                                                              scaleup=up, stride=stride)
                                unpad = rec.get("unpad", (-1, -1))   # (-1, -1): the reference did not resize
                                n = new if isinstance(new, tuple) else (new, new)
                                rows.append([shape[0], shape[1], n[0], n[1], auto, fill, up, stride, unpad[0], unpad[1],
                                             *rec["border"], ratio[0], ratio[1], float(pad[0]), float(pad[1])])
    finally:
        AUG.cv2.resize, AUG.cv2.copyMakeBorder = real_resize, real_border
    return np.array(rows, np.float64)


def main():
    out = {"cv2_version": np.array(cv2.__version__), "geometry": geometry_golden()}
    images = LG.golden_images()
    work = Path(tempfile.mkdtemp(prefix="letterbox_golden_"))
    (work / "images").mkdir()
    (work / "labelTxt").mkdir()
    for i, im in enumerate(images):
        assert cv2.imwrite(str(work / "images" / f"im{i:02d}.png"), im)
        polys = LG.synth_polys(im.shape[0], im.shape[1], 3, 500 + i)
        (work / "labelTxt" / f"im{i:02d}.txt").write_text(
            "".join(" ".join(f"{v:.3f}" for v in p) + " thing 0\n" for p in polys))
    S = LG.GOLDEN_IMG_SIZE
    # detect.py's loader
    for auto in (True, False):
        for i, (_path, img, img0, _cap, _s) in enumerate(D.LoadImages(str(work / "images"), img_size=S, stride=32, auto=auto)):
            assert np.array_equal(img0, images[i])
            out[f"detect/auto{int(auto)}/{i}/shape"], out[f"detect/auto{int(auto)}/{i}/sha256"] = np.array(img.shape), digest(img)
            if auto and i in LG.GOLDEN_FULL_DETECT:
                out[f"detect/auto1/{i}"] = img
    for size in (256, 1024):
        (_path, img, img0, _cap, _s), = list(D.LoadImages(str(REF / "dataset" / "dataset_demo" / "images"), img_size=size))
        out[f"demo/{size}/shape0"] = np.array(img0.shape[:2])
        out[f"demo/{size}/shape"] = np.array(img.shape)
        out[f"demo/{size}/sha256"] = digest(img)
    # val.py's rect loader
    ds = D.LoadImagesAndLabels(str(work / "images"), ClassNames(["thing"]), img_size=S, batch_size=LG.GOLDEN_BATCH, augment=False, hyp=None,
                               rect=True, stride=32, pad=LG.GOLDEN_PAD)
    out["rect/order"] = np.array([int(Path(f).stem[2:]) for f in ds.img_files])
    out["rect/batch_shapes"] = np.array(ds.batch_shapes)
    out["rect/batch"] = np.array(ds.batch)
    for k in range(len(ds)):
        img, labels_out, _f, shapes = ds[k]
        out[f"rect/{k}/shape"], out[f"rect/{k}/sha256"] = np.array(img.shape), digest(img.numpy())
        if int(ds.batch[k]) in LG.GOLDEN_FULL_RECT_BATCHES:
            out[f"rect/{k}/img"] = img.numpy()
        (h0, w0), ((rh, rw), (dw, dh)) = shapes
        out[f"rect/{k}/shapes"] = np.array([h0, w0, rh, rw, dw, dh], np.float64)
        out[f"rect/{k}/rboxes"] = labels_out[:, 1:7].numpy()
    # the reference letterbox on images already in memory, every flag combination that resamples differently
    for i in (0, 2, 6):
        for new, auto, fill, up in ((S, False, True, True), ((96, 160), False, False, False), (160, True, False, True)):
            img, ratio, pad = AUG.letterbox(images[i], new, auto=auto, scaleFill=fill, scaleup=up, stride=32)
            out[f"lb/{i}/{new}/{int(auto)}{int(fill)}{int(up)}/shape"] = np.array(img.shape)
            out[f"lb/{i}/{new}/{int(auto)}{int(fill)}{int(up)}/sha256"] = digest(img)
    np.savez_compressed(HERE / "letterbox_golden.npz", **out)
    print({k: getattr(v, "shape", v) for k, v in out.items()})


if __name__ == "__main__":
    main()
