"""The training loss (csrc/loss.cu through ComputeLoss and autograd) element by element against fp64: items, loss and every
element of the dense gradient, for grad_loss = 1 and 2^16 (a GradScaler scale).  The reference and the per-element bounds are
tests/lossref.py: oracle/loss_ref.py in fp64 with build_targets' decisions in fp32.

Cases: the benchmarked train step (yolov5m b8 1024^2: the Detect logits the train plan produces on bench.train_inputs(8, 0),
TrainStep's hyp), targets on build_targets' boundaries in the 187-, 8- and 7-column layouts, the CloseAug gains (pw 0.825,
anchor_t 3.44), label smoothing, nc = 7, saturated logits, a level without rows, one target, and CIoU ties (equal edges and an
overlap width of exactly 0, where torch's min / max split the derivative and clamp(0) passes it)."""
import time

import pytest
import torch

from tests import lossref
from tests.losscases import FakeModel
from tests.lossgen import exact_cases

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SCALES = (1.0, 2.0 ** 16)


def _check(cl, p, tg, hyp, nc, anchors=lossref.ANCHORS_GRID, strides=lossref.STRIDES):
    t0 = time.perf_counter()
    ref = lossref.reference(p, tg, hyp, nc, anchors, strides)
    bnd = lossref.bounds(p, tg, hyp, nc, anchors, strides)
    pd = [x.detach().to(DEV).float().requires_grad_(True) for x in p]
    loss, items = cl(pd, tg.to(DEV))
    worst = {}
    for gl in SCALES:
        grads = torch.autograd.grad(loss, pd, torch.full_like(loss, gl), retain_graph=True)
        for k, v in lossref.check(grads, loss, items, ref, bnd, gl).items():
            worst[k] = max(worst.get(k, 0.0), v)
    torch.cuda.synchronize()
    return bnd, worst, time.perf_counter() - t0


def _report(name, bnd, worst, sec):
    w = ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items()))
    print(f"\n{name}: rows per level {bnd['nrows']}; worst error / bound: {w}; {sec:.1f} s")


@pytest.mark.parametrize("name", sorted(exact_cases()))
def test_case(name):
    from yolov5_obb_b200.loss import ComputeLoss
    p, tg, hyp, nc = exact_cases()[name]()
    cl = ComputeLoss(FakeModel(hyp, nc=nc))
    bnd, worst, sec = _check(cl, p, tg, hyp, nc)
    _report(name, bnd, worst, sec)
    if name == "p5-no-rows":
        assert bnd["nrows"][2] == 0


def test_benchmarked_step():
    """yolov5m b8 1024^2: the logits the train plan itself produces for bench.train_inputs(8, 0), and the hyp of
    TrainStep(m, batch_size=64, imgsz=1024, warmup_iters=1000), as bench.py's train leg builds them."""
    import bench
    from tests.modelgen import build_mirror
    from yolov5_obb_b200.train_step import TrainStep
    m = build_mirror(bench.TRAIN_MODEL, nc=bench.NC, seed=0).train().to(DEV)
    ts = TrainStep(m, batch_size=64, imgsz=bench.IMG, warmup_iters=1000)
    imgs, tg = bench.train_inputs(bench.TRAIN_BATCH, 0)
    assert tg.shape[0] == bench.TRAIN_BATCH * bench.TRAIN_TARGETS_PER_IMG
    pred = m(imgs.to(DEV))
    p = [x.detach().float().cpu() for x in pred]
    det = m.model[-1]
    anchors = det.anchors.detach().float().cpu()
    strides = [float(s) for s in det.stride]
    bnd, worst, sec = _check(ts.compute_loss, p, tg, ts.hyp, det.nc, anchors, strides)
    _report("yolov5m b8 1024x1024 train step", bnd, worst, sec)
    assert sum(bnd["nrows"]) > 0
