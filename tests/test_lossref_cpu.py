"""CPU checks of tests/lossref.py: the reference's own fp32 arithmetic (oracle/loss_ref.py in fp32, autograd gradients) stays
under a quarter of every per-element bound against the fp64 reference, on >= 10^5 random rows and on every edge case the GPU
test runs.  This shows the bounds the kernel is held to are achievable by correct fp32 code."""
import pytest
import torch

from oracle import loss_ref
from tests import lossref
from tests.losscases import ANCHORS_GRID, STRIDES
from tests.lossgen import exact_cases, synth_preds, synth_targets


def _fp32_run(p, tg, hyp, nc):
    p32 = [x.detach().clone().float().requires_grad_(True) for x in p]
    with lossref.serial():
        loss, items = loss_ref.compute_loss(p32, lossref.expand_csl(tg), ANCHORS_GRID, STRIDES, hyp, nc)
    loss.backward()
    return [x.grad for x in p32], loss.detach(), items


def _check_fp32(p, tg, hyp, nc):
    ref = lossref.reference(p, tg, hyp, nc)
    bnd = lossref.bounds(p, tg, hyp, nc)
    grads, loss, items = _fp32_run(p, tg, hyp, nc)
    worst = lossref.check(grads, loss, items, ref, bnd)
    assert max(worst.values()) <= 0.25, str(worst)
    return ref, bnd, worst


def test_loss_ref_keeps_fp64():
    p = synth_preds(2, 128, seed=1)
    tg = torch.from_numpy(synth_targets(2, 12, 128, seed=1))
    hyp = loss_ref.scaled_hyp(loss_ref.DEFAULT_HYP, 3, 15, 128)
    loss, items = loss_ref.compute_loss([x.double() for x in p], tg, ANCHORS_GRID, STRIDES, hyp, 15)
    assert loss.dtype == items.dtype == torch.float64


def test_random_rows():
    """~1.2 10^5 matched rows on a 2 x 256^2 input: most cells take several rows (the atomics' count term)."""
    hyp = loss_ref.scaled_hyp(loss_ref.DEFAULT_HYP, 3, 15, 256)
    p = synth_preds(2, 256, seed=21)
    tg = torch.from_numpy(synth_targets(2, 16000, 256, seed=21))
    _, bnd, worst = _check_fp32(p, tg, hyp, 15)
    assert sum(bnd["nrows"]) >= 10 ** 5
    print(f"\nrandom rows {sum(bnd['nrows'])}: worst fp32 error / bound {worst}")


@pytest.mark.parametrize("name", sorted(exact_cases()))
def test_edge_cases(name):
    p, tg, hyp, nc = exact_cases()[name]()
    _, bnd, worst = _check_fp32(p, tg, hyp, nc)
    print(f"\n{name}: rows per level {bnd['nrows']}, worst fp32 error / bound {worst}")
    if name == "p5-no-rows":
        assert bnd["nrows"][2] == 0 and bnd["nrows"][0] > 0
    if name == "nt1":
        assert tg.shape[0] == 1 and sum(bnd["nrows"]) > 0


def test_boundary_targets_reach_the_decisions():
    """The boundary rows do reach each decision: negative-CIoU winners, clamped cells with an unclamped tbox, and the
    anchor-ratio rows at exactly anchor_t rejected."""
    p, tg, hyp, nc = exact_cases()["boundary-187"]()
    tcls, tbox, indices, anch, _ = loss_ref.build_targets(p, tg, ANCHORS_GRID, STRIDES, hyp["anchor_t"], 3)
    b, a, gj, gi = indices[0]
    W0 = p[0].shape[3]
    assert bool(((gi == W0 - 1) & (tbox[0][:, 0] < 1)).any())    # clamped from W: tx = gx - W (unclamped) = 0
    assert bool(((gi == 0) & (tbox[0][:, 0] < 0)).any())         # clamped from -1
    ciou = lossref._ciou_rows(p[0].double()[b, a, gj, gi], tbox[0], anch[0])[0]
    assert bool((ciou < 0).any()) and bool((ciou > 0).any())
    r = tbox[0][:, 2] / anch[0][:, 0]
    assert not bool((torch.max(r, 1 / r) == 4.0).any())          # the l / anchor == 4.0 row is rejected
