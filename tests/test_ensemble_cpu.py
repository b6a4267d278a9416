"""CPU checks of model ensembles (yolov5_obb_b200.ensemble, engine.ensemble_layout): the attributes attempt_load gives an
ensemble (models/experimental.py:112-120), the row layout of the concatenated output computed from shapes alone, and the
refusals.  Nothing here runs a kernel."""
import pytest
import torch

from tests.modelgen import build_mirror
from yolov5_obb_b200.engine import EnsemblePlan, ensemble_layout, tta_geometry
from yolov5_obb_b200.ensemble import Ensemble, attempt_load


def _member(key, nc=15, names=None):
    m = build_mirror(key, nc=nc, seed=0)
    if names is not None:
        m.names = names
    return m


def _ref_attrs(models):
    """experimental.py:118-119 restated: names of the last member, the stride tensor of the member with the largest max
    stride (torch.argmax: the first one)."""
    i = int(torch.argmax(torch.tensor([m.stride.max() for m in models])))
    return models[-1].names, models[i].stride


@pytest.mark.parametrize("keys", [("n", "s"), ("n", "n6"), ("n6", "n"), ("s6", "n6", "n"), ("n", "s", "m")])
def test_attributes_follow_attempt_load(keys):
    models = [_member(k, names=[f"{k}-{c}" for c in range(15)]) for k in keys]
    ens = attempt_load(models)
    assert isinstance(ens, Ensemble) and len(ens) == len(models) and list(ens) == models
    names, stride = _ref_attrs(models)
    assert ens.names == names and ens.names[0] == f"{keys[-1]}-0"
    assert ens.stride is stride
    assert [float(s) for s in ens.stride] == ([8.0, 16.0, 32.0, 64.0] if any(k.endswith("6") for k in keys)
                                              else [8.0, 16.0, 32.0])
    assert ens.nc == 15 and not ens.training


def test_single_member_is_the_model_itself():
    m = _member("n")
    assert attempt_load([m]) is m
    assert attempt_load(m) is m


# n (P5) and n6 (P6) at 256 x 320, counted by hand: plain rows 3 * sum(H/s * W/s) per member; with augment=True each
# member's own _forward_augment branches
P5_PLAIN = 3 * (32 * 40 + 16 * 20 + 8 * 10)                    # 5040
P6_PLAIN = P5_PLAIN + 3 * (4 * 5)                              # 5100
P5_TTA = 3 * (32 * 40 + 16 * 20) + 3 * (28 * 36 + 14 * 18 + 7 * 9) + 3 * (12 * 14 + 6 * 7)
#        scale 1 (levels 0, 1)     0.83 -> 224 x 288 (all levels)     0.67 -> 192 x 224 (levels 1, 2)
P6_TTA = 3 * (32 * 40 + 16 * 20 + 8 * 10) + P6_PLAIN + 3 * (12 * 16 + 6 * 8 + 3 * 4)
#        scale 1 (levels 0-2)               0.83 -> 256 x 320   0.67 -> 192 x 256 (levels 1-3)


def test_row_layout_plain_and_tta():
    n, n6 = _member("n"), _member("n6")
    assert ensemble_layout([n, n6], 256, 320) == ([0, P5_PLAIN], P5_PLAIN + P6_PLAIN)
    assert ensemble_layout([n6, n], 256, 320) == ([0, P6_PLAIN], P5_PLAIN + P6_PLAIN)
    assert ensemble_layout([n, n, n], 256, 320) == ([0, P5_PLAIN, 2 * P5_PLAIN], 3 * P5_PLAIN)
    # test-time augmentation: each member pads its branches to its OWN largest stride, so the P5 member's rows at a size
    # that is a multiple of 64 are those it has alone, not those of a stride-64 padding
    assert P5_TTA == 9399 and P6_TTA == 10896
    assert tta_geometry(256, 320, 32)[1] == P5_TTA
    assert tta_geometry(256, 320, 64, 4, 3, [8, 16, 32, 64])[1] == P6_TTA
    assert tta_geometry(256, 320, 64)[1] != P5_TTA                  # (a shared gs would change the P5 member's rows)
    assert ensemble_layout([n, n6], 256, 320, augment=True) == ([0, P5_TTA], P5_TTA + P6_TTA)
    assert ensemble_layout([n6, n], 256, 320, augment=True) == ([0, P6_TTA], P5_TTA + P6_TTA)
    # a P5-only ensemble keeps the stride-32 sizes
    assert ensemble_layout([n, n], 96, 160)[1] == 2 * 3 * (12 * 20 + 6 * 10 + 3 * 5)
    assert ensemble_layout([n, n], 96, 160, augment=True) == ([0, tta_geometry(96, 160)[1]], 2 * tta_geometry(96, 160)[1])


def test_row_layout_refuses_sizes_off_the_largest_stride():
    n, n6 = _member("n"), _member("n6")
    for aug in (False, True):
        with pytest.raises(RuntimeError, match="largest stride 64"):
            ensemble_layout([n, n6], 224, 320, augment=aug)
    ensemble_layout([n, n], 224, 320)


def test_refusals():
    n = _member("n")
    with pytest.raises(RuntimeError, match="at least one"):
        Ensemble([])
    with pytest.raises(RuntimeError, match="at least one"):
        attempt_load([])
    with pytest.raises(RuntimeError, match="class counts"):
        Ensemble([n, _member("n", nc=16)])
    with pytest.raises(RuntimeError, match="different devices"):
        Ensemble([n, _member("n").to("meta")])
    t = _member("n").train()
    with pytest.raises(RuntimeError, match="eval mode"):
        Ensemble([n, t])
    ens = Ensemble([n, _member("n6")])
    with pytest.raises(RuntimeError, match="inference"):
        ens.train()
    ens.eval()                                   # eval() stays allowed
    n.train()
    try:                                         # a member switched to training after the ensemble was built
        with pytest.raises(RuntimeError, match="eval mode"):
            ens.records_plan((1, 3, 64, 64), "cpu")
    finally:
        n.eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        EnsemblePlan(list(ens), 1, 64, 64, "cpu")
    from yolov5_obb_b200.val import Validator
    with pytest.raises(RuntimeError, match="ensemble"):
        Validator(ens, compute_loss=object())
