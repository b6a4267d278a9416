"""GPU: y5obb_augment_images_u8 / y5obb_augment_labels against the REFERENCE's __getitem__ + collate_fn (augment_golden.npz)
and against the numpy restatement (oracle/augment_ref.py) at training scale; edge cases, refusals, and the loader feeding
TrainStep."""
import copy

import numpy as np
import pytest
import torch

from oracle import augment_ref as A
from tests.augmentgen import HYP_DOTA, synth_dataset
from tests.test_augment_cpu import CASES, G, S, assert_rows_close, replay
from yolov5_obb_b200 import augment as P

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def oracle_rows(recs, labels, S, hyp):
    rows = []
    for b, r in enumerate(recs):
        t = A.targets_from_polys(A.sample_polys(r, labels, S), S, hyp["cls_theta"], hyp["csl_radius"])
        rows.append(np.concatenate([np.full((len(t), 1), b, np.float32), t], 1))
    return np.concatenate(rows)


def check_rows(got, want):
    """Device rows against the oracle's: the same rows in the same order; the rbox columns are poly2rbox in fp64 on both
    sides (the device's minAreaRect restatement agrees with the oracle's to 1e-9), so they agree to fp32 rounding; the CSL
    rows agree wherever the angle is not within rounding of a bin edge."""
    assert got.shape == want.shape, (got.shape, want.shape)
    assert np.array_equal(got[:, :2], want[:, :2])
    np.testing.assert_allclose(got[:, 2:7], want[:, 2:7], rtol=2e-7, atol=1e-5)
    ang = want[:, 6].astype(np.float64) * 180 / 3.141592 + 90
    safe = np.abs(ang - np.round(ang)) > 1e-3
    np.testing.assert_allclose(got[safe, 7:], want[safe, 7:], rtol=0, atol=1e-7)


@pytest.mark.parametrize("name", CASES)
def test_device_matches_reference_goldens(name):
    images, labels, hyp, batches = replay(name)
    ds = P.DeviceDataset(images, labels, S, DEV)
    for k, idx, recs in batches:
        imgs, tg = P.augment_batch(ds, recs, 187, hyp["cls_theta"], hyp["csl_radius"])
        assert imgs.dtype == torch.uint8 and imgs.shape == (len(idx), 3, S, S)
        assert torch.equal(imgs.cpu(), torch.from_numpy(G[f"{name}/{k}/imgs"])), name
        got, want = tg.cpu().numpy(), G[f"{name}/{k}/targets"]
        assert got.shape == want.shape and np.array_equal(got[:, :2], want[:, :2])
        assert_rows_close(got, want)
        check_rows(got, oracle_rows(recs, labels, S, hyp))
        _, tc = P.augment_batch(ds, recs, 8, hyp["cls_theta"], hyp["csl_radius"])
        tc = tc.cpu().numpy()
        assert np.array_equal(tc[:, :7], got[:, :7])
        # column 7 = int(90 - angle): the CSL row of the full form peaks at bin (90 - index) mod 180
        assert np.array_equal((90 - tc[:, 7]) % 180, got[:, 7:].argmax(1))


def test_device_matches_oracle_at_scale():
    """S = 1024, B = 16, up to 150 labels per image, dota's probabilities with mixup forced on a share of the samples."""
    S1, B = 1024, 16
    images, labels = synth_dataset(24, S1, 7, max_labels=150)
    hyp = dict(HYP_DOTA, mixup=0.5)
    import random
    random.seed(11)
    np.random.seed(11)
    ds = P.DeviceDataset(images, labels, S1, DEV)
    recs = P.plan_batch(ds, range(B), hyp)
    imgs, tg = P.augment_batch(ds, recs, 187, 180, hyp["csl_radius"])
    got = imgs.cpu().numpy()
    for b, r in enumerate(recs):
        want = A.sample_image(r, images, S1)[:, :, ::-1].transpose(2, 0, 1)
        assert np.array_equal(got[b], want), (b, int((got[b] != want).sum()))
    assert any(r["mix_r"] is not None for r in recs) and any(len(r["groups"][0]["img"]) == 1 for r in recs)
    want = oracle_rows(recs, labels, S1, hyp)
    assert len(want) > 500
    check_rows(tg.cpu().numpy(), want)


def test_empty_and_all_filtered_labels():
    images, labels = synth_dataset(6, 128, 5)
    hyp = dict(HYP_DOTA, mosaic=1.0)
    import random
    for lab in ([np.zeros((0, 9), np.float32)] * 6,
                [np.array([[1, -5e3, -5e3, -4e3, -5e3, -4e3, -4e3, -5e3, -4e3]], np.float32)] * 6):
        ds = P.DeviceDataset(images, lab, 128, DEV)
        random.seed(0)
        np.random.seed(0)
        recs = P.plan_batch(ds, [0, 1, 2], hyp)
        for tcols in (187, 8):
            imgs, tg = P.augment_batch(ds, recs, tcols, 180, hyp["csl_radius"])
            assert tg.shape == (0, tcols)
            assert torch.equal(imgs.cpu(), torch.from_numpy(np.stack(
                [A.sample_image(r, images, 128)[:, :, ::-1].transpose(2, 0, 1) for r in recs])))


def test_refusals():
    from yolov5_obb_b200 import _lib
    images, labels = synth_dataset(4, 128, 1)
    with pytest.raises(ValueError):
        P.DeviceDataset(images, labels, 96 + 1, DEV)          # S not a multiple of 32
    with pytest.raises(ValueError):
        P.DeviceDataset(images, labels, 96, DEV)              # images over img_size
    ds = P.DeviceDataset(images, labels, 128, DEV)
    import random
    random.seed(0)
    np.random.seed(0)
    recs = P.plan_batch(ds, [0, 1], dict(HYP_DOTA, mosaic=1.0))
    bad = copy.deepcopy(recs)
    bad[1]["groups"][0]["img"][2] = 99                         # bad id
    with pytest.raises(RuntimeError):
        P.augment_batch(ds, bad)
    bad = copy.deepcopy(recs)
    bad[0]["groups"][0]["pad"][0] = (-300, 0)                  # placement outside its image
    with pytest.raises(RuntimeError):
        P.augment_batch(ds, bad)
    with pytest.raises(ValueError):
        P.augment_batch(ds, recs, tcols=20)
    # the C entry: an image over S, and label rows outside the label buffer
    meta = ds.meta_host.copy()
    recs_c = (P.SampleRec * 2)(*[P.pack_record(r) for r in recs])
    import ctypes
    L = _lib.lib()
    args = lambda m, nl: (m.ctypes.data, ds.n, ds.images.numel(), nl, ctypes.addressof(recs_c), 2, 128)
    assert L.y5obb_augment_check(*args(meta, ds.labels.numel() // 9)) == 0
    m2 = meta.copy()
    m2[0, 1] = 160
    assert L.y5obb_augment_check(*args(m2, ds.labels.numel() // 9)) == 1
    assert L.y5obb_augment_check(*args(meta, ds.labels.numel() // 9 - 1)) == 1
    assert L.y5obb_augment_check(meta.ctypes.data, ds.n, ds.images.numel(), ds.labels.numel() // 9,
                                 ctypes.addressof(recs_c), 2, 120) == 1


def test_loader_batch_feeds_train_step():
    """A loader batch fed to TrainStep.step gives the same loss as the same batch uploaded from the host; the loader is
    deterministic for a seed."""
    from tests.modelgen import build_mirror
    from yolov5_obb_b200.train_step import TrainStep
    images, labels = synth_dataset(10, 128, 9)
    ds = P.DeviceDataset(images, labels, 128, DEV)
    hyp = dict(HYP_DOTA)

    def first_batches(n):
        out = []
        for imgs, tg in P.DeviceAugmentLoader(ds, hyp, batch_size=4, shuffle=True, seed=5):
            out.append((imgs.clone(), tg.clone()))
            if len(out) == n:
                break
        return out

    a, b = first_batches(3), first_batches(3)
    for (ia, ta), (ib, tb) in zip(a, b):
        assert torch.equal(ia, ib) and torch.equal(ta, tb)
    loader = P.DeviceAugmentLoader(ds, hyp, batch_size=4, shuffle=True, seed=5)
    assert len(loader) == 3
    m = build_mirror("n", nc=15, seed=0, obj_bias=1.0, cls_bias=-1.0, det_gain=6.0)
    m1, m2 = copy.deepcopy(m).to(DEV).train(), copy.deepcopy(m).to(DEV).train()
    t1 = TrainStep(m1, batch_size=4, imgsz=128)
    t2 = TrainStep(m2, batch_size=4, imgsz=128)
    imgs, tg = next(iter(loader))
    assert tg.shape[1] == 187 and tg.shape[0] > 0
    host_imgs, host_tg = imgs.cpu().pin_memory(), tg.cpu().pin_memory()
    l1, _ = t1.step(imgs, tg)
    l2, _ = t2.step(host_imgs.to(DEV), host_tg.to(DEV))
    torch.cuda.synchronize()
    assert torch.isfinite(l1).all() and torch.equal(l1, l2)
