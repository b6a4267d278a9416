"""Goldens for the training augmentation from the REFERENCE's own LoadImagesAndLabels.__getitem__ (utils/datasets.py:561-665)
and collate_fn (:668-672), run on a stand-in dataset object holding the cached synthetic set of tests/augmentgen.py
(opencv-python 4.13.0 when they were made).  The fp32 polygons __getitem__ hands to poly2rbox are recorded as well.
python tests/golden/make_augment_golden.py"""
import json
import random
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import ref_import  # noqa: E402

ref_import.setup()
sys.path.insert(0, str(HERE.parents[1]))
import utils.datasets as D  # noqa: E402
from tests.augmentgen import HYP_DOTA, synth_dataset  # noqa: E402

S, N_IMAGES, DATA_SEED = 128, 12, 3
# (name, hyp overrides, seed, batches of indices): each forces a branch of __getitem__
CASES = [
    ("dota", {}, 0, [[0, 1, 2, 3], [4, 5, 6, 7]]),
    ("mosaic_only", dict(mosaic=1.0, mixup=0.0, flipud=0.0, fliplr=0.0), 1, [[8, 9, 10, 11]]),
    ("letterbox", dict(mosaic=0.0, flipud=0.0, fliplr=0.0), 2, [[0, 1, 2, 3, 4, 5]]),
    ("mixup_flips", dict(mosaic=1.0, mixup=1.0, flipud=1.0, fliplr=1.0), 3, [[4, 9, 1, 6]]),
    ("letterbox_flips_nohsv", dict(mosaic=0.0, flipud=1.0, fliplr=1.0, hsv_h=0.0, hsv_s=0.0, hsv_v=0.0), 4, [[7, 2, 11]]),
]


class Stand:
    """The attributes __getitem__ / load_mosaic / load_image_label read, for a set cached in RAM (augment=True, rect=False)."""

    def __init__(self, images, labels, hyp):
        self.img_size, self.augment, self.rect, self.mosaic, self.hyp = S, True, False, True, hyp
        self.mosaic_border = [-S // 2, -S // 2]
        self.n = len(images)
        self.indices = range(self.n)
        self.imgs = images
        self.img_hw0 = self.img_hw = [im.shape[:2] for im in images]
        self.labels = labels
        self.segments = [[] for _ in images]
        self.img_files = [f"synth{i}.png" for i in range(self.n)]

    __getitem__ = D.LoadImagesAndLabels.__getitem__


def main():
    import cv2
    images, labels = synth_dataset(N_IMAGES, S, DATA_SEED)
    seen = []
    orig = D.poly2rbox

    def rec(polys, **kw):
        seen.append(np.asarray(polys, np.float32).copy())
        return orig(polys=polys, **kw)

    D.poly2rbox = rec
    out = {"cv2_version": np.array(cv2.__version__), "S": np.array(S), "n_images": np.array(N_IMAGES),
           "data_seed": np.array(DATA_SEED)}
    for name, over, seed, batches in CASES:
        hyp = dict(HYP_DOTA, **over)
        ds = Stand(images, labels, hyp)
        random.seed(seed)
        np.random.seed(seed)
        for k, idx in enumerate(batches):
            items = []
            for i in idx:
                del seen[:]
                img, lab, path, shapes = ds[i]
                items.append((img, lab, path, shapes))
                out[f"{name}/{k}/polys{len(items) - 1}"] = seen[0] if seen else np.zeros((0, 8), np.float32)
            imgs, tg, _, _ = D.LoadImagesAndLabels.collate_fn(items)
            out[f"{name}/{k}/idx"] = np.array(idx)
            out[f"{name}/{k}/imgs"] = imgs.numpy()
            out[f"{name}/{k}/targets"] = tg.numpy()
        out[f"{name}/seed"] = np.array(seed)
        out[f"{name}/hyp"] = np.array(json.dumps(hyp))
    np.savez_compressed(HERE / "augment_golden.npz", **out)
    print({k: getattr(v, "shape", v) for k, v in out.items() if k.endswith("targets")})


if __name__ == "__main__":
    main()
