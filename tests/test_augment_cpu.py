"""CPU: the host plan (yolov5_obb_b200/augment.py) and the numpy restatement (oracle/augment_ref.py) against the REFERENCE's
own __getitem__ + collate_fn outputs (augment_golden.npz), and each restated cv2 operation against cv2 where it imports."""
import json
import random
from pathlib import Path

import numpy as np
import pytest

from oracle import augment_ref as A
from tests.augmentgen import synth_dataset
from yolov5_obb_b200 import augment as P

G = np.load(Path(__file__).resolve().parent / "golden" / "augment_golden.npz")
S = int(G["S"])
CASES = sorted({k.split("/")[0] for k in G.files if "/" in k})


def golden_batches(name):
    k = 0
    while f"{name}/{k}/idx" in G.files:
        yield k, G[f"{name}/{k}/idx"]
        k += 1


def replay(name):
    """The plans of a golden case: the same seeds, the same indices, the host plan's draws."""
    images, labels = synth_dataset(int(G["n_images"]), S, int(G["data_seed"]))
    hyp = json.loads(str(G[f"{name}/hyp"]))
    random.seed(int(G[f"{name}/seed"]))
    np.random.seed(int(G[f"{name}/seed"]))
    shapes = [im.shape[:2] for im in images]
    out = []
    for k, idx in golden_batches(name):
        out.append((k, idx, [P.plan_sample(int(i), len(images), shapes, S, hyp) for i in idx]))
    return images, labels, hyp, out


@pytest.mark.parametrize("name", CASES)
def test_plan_and_oracle_reproduce_reference_getitem(name):
    images, labels, hyp, batches = replay(name)
    for k, idx, recs in batches:
        imgs = np.stack([A.sample_image(r, images, S)[:, :, ::-1].transpose(2, 0, 1) for r in recs])
        assert np.array_equal(imgs, G[f"{name}/{k}/imgs"]), (name, k, int((imgs != G[f"{name}/{k}/imgs"]).sum()))
        rows = []
        for b, r in enumerate(recs):
            L = A.sample_polys(r, labels, S)
            want = G[f"{name}/{k}/polys{b}"]
            assert np.array_equal(L[:, 1:], want.reshape(-1, 8)), (name, k, b)
            t = A.targets_from_polys(L, S, hyp["cls_theta"], hyp["csl_radius"])
            rows.append(np.concatenate([np.full((len(t), 1), b, np.float32), t], 1))
        got, want = np.concatenate(rows), G[f"{name}/{k}/targets"]
        assert got.shape == want.shape
        assert np.array_equal(got[:, :2], want[:, :2])
        assert_rows_close(got, want)


def assert_rows_close(got, want):
    """poly2rbox is cv2.minAreaRect, restated in fp64 (oracle/rbox_ref.py, tests/test_oracle_p2r.py): rows agree except
    where cv2's float32 arithmetic decides a near-tie between hull edges (thin and degenerate boxes), as in
    tests/test_rbox_gpu.py"""
    d = np.abs(got[:, 2:6] - want[:, 2:6]).max(1)
    assert (d > 2e-3).mean() <= 0.15, d


def test_branches_are_covered():
    flags = set()
    for name in CASES:
        for _, _, recs in replay(name)[3]:
            for r in recs:
                flags |= {("mosaic", len(r["groups"][0]["img"]) == 4), ("mixup", r["mix_r"] is not None),
                          ("hsv", r["luts"] is not None), ("flipud", r["flipud"]), ("fliplr", r["fliplr"])}
    assert flags == {(a, v) for a in ("mosaic", "mixup", "hsv", "flipud", "fliplr") for v in (False, True)}


def test_plan_refuses_perspective():
    images, labels = synth_dataset(4, 64, 0)
    hyp = json.loads(str(G["dota/hyp"]))
    hyp["perspective"] = 1e-4
    with pytest.raises(ValueError):
        P.plan_sample(0, 4, [im.shape[:2] for im in images], 64, dict(hyp, mosaic=1.0))


cv2 = pytest.importorskip("cv2")


def test_rotation_and_inverse_match_cv2():
    rng = np.random.default_rng(0)
    for _ in range(200):
        a, s = rng.uniform(-180, 180), rng.uniform(0.5, 1.5)
        assert np.array_equal(P.rotation_matrix_2d(a, s), cv2.getRotationMatrix2D(angle=a, center=(0, 0), scale=s))
        M = rng.normal(size=(2, 3)) * [1, 1, 200]
        assert np.array_equal(P.invert_affine(M), cv2.invertAffineTransform(M).reshape(-1))


def test_warp_affine_matches_cv2():
    rng = np.random.default_rng(1)
    src = rng.integers(0, 256, (300, 400, 3), dtype=np.uint8)
    for t in range(6):
        R = np.eye(3)
        R[:2] = cv2.getRotationMatrix2D(angle=rng.uniform(-180, 180), center=(0, 0), scale=rng.uniform(0.6, 1.4))
        T = np.eye(3)
        T[:2, 2] = rng.uniform(-50, 300, 2)
        C = np.eye(3)
        C[:2, 2] = [-200, -150]
        M = (T @ R @ C)[:2]
        want = cv2.warpAffine(src, M, dsize=(256, 256), borderValue=(114, 114, 114))
        got = A.warp_affine_u8(src, P.invert_affine(M), 256, 256)
        assert np.array_equal(got, want), (t, int((got != want).sum()))


def test_bgr2hsv_all_colours():
    v = np.arange(1 << 24, dtype=np.uint32)
    bgr = np.stack([v & 255, (v >> 8) & 255, v >> 16], -1).astype(np.uint8).reshape(4096, 4096, 3)
    assert np.array_equal(A.bgr2hsv_u8(bgr), cv2.cvtColor(bgr, cv2.COLOR_BGR2HSV))


def test_hsv2bgr_all_triples():
    h, s, v = np.meshgrid(np.arange(180), np.arange(256), np.arange(256), indexing="ij")
    hsv = np.stack([h, s, v], -1).astype(np.uint8).reshape(180 * 256, 256, 3)   # rows of 256: cv2's vector loop
    assert np.array_equal(A.hsv2bgr_u8(hsv), cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR))
