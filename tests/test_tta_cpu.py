"""CPU tests of test-time augmentation: the fp32 oracle's forward_augment (oracle/tta_ref.py) against the REFERENCE model's own
`m(x, augment=True)` (tests/golden/tta_golden.npz, made by make_tta_golden.py, laid out as tests/ttagen.py describes: every
row's box columns, every column of sampled rows, every row's sum), and the host geometry of the device plan
(engine.tta_geometry) against the reference's scale_img / _clip_augmented arithmetic for every multiple-of-32 shape up to 2048."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import tta_ref
from tests.modelgen import build_mirror
from tests.ttagen import pieces, tta_input
from yolov5_obb_b200.engine import tta_geometry

ROOT = Path(__file__).resolve().parents[1]
G = np.load(ROOT / "tests" / "golden" / "tta_golden.npz")


@pytest.mark.parametrize("size", ["n", "s"])
def test_oracle_forward_augment_matches_reference(size):
    m = build_mirror(size, nc=15, seed=0)
    x = tta_input()
    assert x.double().sum().item() == float(G["x_sum"])
    pred, none = tta_ref.forward_augment(m, x)
    branches, rows = tta_geometry(128, 160)
    assert none is None and tuple(pred.shape) == tuple(G[f"{size}/shape"]) == (2, rows, 200)
    got = pieces(pred.numpy())
    for k in ("box", "rows"):
        assert np.abs(got[k] - G[f"{size}/{k}"]).max() < 1e-5, k
    # every element, through its row's sum: each of the 200 terms within the same bound
    assert np.abs(got["rowsum"] - G[f"{size}/rowsum"]).max() < 200 * 1e-5


def test_geometry_of_the_golden_shape():
    branches, rows = tta_geometry(128, 160)
    assert [(b["h"], b["w"], b["Hp"], b["Wp"]) for b in branches] == [(128, 160, 128, 160), (106, 132, 128, 160), (85, 107, 96, 128)]
    assert [b["levels"] for b in branches] == [(0, 1), (0, 1, 2), (1, 2)]
    assert rows == 2640


def test_geometry_at_1024():
    branches, rows = tta_geometry(1024, 1024)
    assert [(b["h"], b["Hp"]) for b in branches] == [(1024, 1024), (849, 864), (686, 704)]
    assert [b["rows"] for b in branches] == [61440, 45927, 7260] and rows == 114627
    assert [b["row_off"] for b in branches] == [0, 61440, 61440 + 45927]
    assert branches[1]["flip"] == 3 and branches[1]["flip_w"] == 1024.0 and branches[2]["flip_w"] == 0.0
    assert branches[1]["inv_scale"] == float(np.float32(1.0) / np.float32(0.83))


def _reference_rows(H, W, na=3, strides=(8, 16, 32)):
    """scale_img's output shape (on the meta device, the reference's own F.interpolate / F.pad size arithmetic), then
    _clip_augmented applied to row ids: the ids each branch keeps."""
    ids = []
    for s, f in zip(tta_ref.SCALES, tta_ref.FLIPS):
        xi = tta_ref.scale_img(torch.empty(1, 3, H, W, device="meta"), s, gs=32)
        Hp, Wp = xi.shape[2:]
        n = sum(na * (Hp // st) * (Wp // st) for st in strides)
        ids.append((torch.arange(n).view(1, n, 1), (Hp, Wp)))
    kept = tta_ref.clip_augmented([t for t, _ in ids])
    return [(k[0, :, 0], hw) for k, (_, hw) in zip(kept, ids)]


def test_geometry_equals_reference_arithmetic_for_every_multiple_of_32():
    sizes = range(32, 2049, 32)
    for H in sizes:
        for W in sizes:
            branches, rows = tta_geometry(H, W)
            ref = _reference_rows(H, W)
            total = 0
            for b, (kept, (Hp, Wp)) in zip(branches, ref):
                assert (b["Hp"], b["Wp"]) == (Hp, Wp), (H, W)
                # the kept row ids are exactly the kept Detect levels, in order
                starts = np.cumsum([0] + b["level_rows"])
                want = torch.cat([torch.arange(int(starts[l]), int(starts[l + 1])) for l in b["levels"]])
                assert torch.equal(kept, want), (H, W, b["scale"])
                assert b["rows"] == kept.numel() and b["row_off"] == total
                total += b["rows"]
            assert rows == total
    with pytest.raises(RuntimeError):
        tta_geometry(72, 64)
