"""The compact-record Detect epilogue (epilogue_records in conv_sm90.cu) against the shared epilogue it replaces
(Y5OBB_CONV_DETECT_GENERIC), byte for byte, on every Detect launch of a plan.

Both arms run the same plan on the same input and write into sentinel-filled record buffers that are wider than the
region the plan writes (rows before and after it), so the padding columns of every record and every byte outside the
region are compared too.  The calibrated benchmark model gives the theta logits real near-ties.  The plans cover the
benchmark's, a wider model, four Detect levels, the de-scaled and flipped TTA branches, tiles narrower than the image
(Wt != Wout, ragged right and bottom edges: 1056^2, 1024 x 768 letterboxed) and a batch of one."""
import functools

import pytest
import torch

import bench
from tests.modelgen import calibrated_bench_model
from yolov5_obb_b200.conv import DETECT_GENERIC
from yolov5_obb_b200.engine import InferenceEngine, TTAPlan

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SENTINEL = 0x7FC0DEAD   # a NaN payload no record holds
PAD_ROWS = 37           # rows of sentinel before and after the plan's region


@functools.lru_cache(maxsize=None)
def _model(size, nc=bench.NC):
    return calibrated_bench_model(size, nc=nc, seed=0, conf=bench.CONF).to(DEV)


def _batch(B, H, W, seed):
    if (H, W) == (bench.IMG, bench.IMG):
        return bench.synth_batch(B, seed).to(DEV)
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, generator=g).to(DEV)


def _sentinel(shape):
    return torch.full(shape, SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)


def _compare(a, b, what):
    ai, bi = a.view(torch.int32), b.view(torch.int32)
    if not torch.equal(ai, bi):
        bad = (ai != bi).nonzero()
        raise AssertionError(f"{what}: {bad.shape[0]} words differ, first at {bad[0].tolist()}: "
                             f"{a[tuple(bad[0])].item()!r} vs {b[tuple(bad[0])].item()!r}")


def _records(size, B, H, W, seed=0, nc=bench.NC):
    m = _model(size, nc)
    x = _batch(B, H, W, seed)
    probe = InferenceEngine(m, B, H, W, DEV, compact_detect=True)
    rows, rec_w = probe.rows_total, probe.rec_w
    del probe
    outs = []
    for flags in (0, DETECT_GENERIC):
        buf = _sentinel((B, PAD_ROWS + rows + PAD_ROWS, rec_w))
        eng = InferenceEngine(m, B, H, W, DEV, conv_flags=flags, compact_detect=True, det_out=buf, det_row_base=PAD_ROWS)
        eng.forward(x)
        torch.cuda.synchronize()
        outs.append(buf)
        del eng
    new, old = outs
    region = old[:, PAD_ROWS:PAD_ROWS + rows]
    assert not torch.isnan(region).any(), "the generic epilogue left rows of the region unwritten"
    outside = torch.cat([old[:, :PAD_ROWS], old[:, PAD_ROWS + rows:]], 1).view(torch.int32)
    assert bool((outside == SENTINEL).all()), "the generic epilogue wrote outside the region"
    _compare(new, old, f"yolov5{size} B{B} {H}x{W}")
    th = region[..., 5 + m.model[-1].nc]
    return th


@pytest.mark.parametrize("size,B,H,W", [
    ("s", 16, 1024, 1024),   # the benchmark's plan
    ("m", 16, 1024, 1024),
    ("s6", 4, 1280, 1280),   # four Detect levels
    ("s", 2, 1056, 1056),    # the whole-scene tile: Wt = 16 on a 132-wide P3 grid, ragged right and bottom tiles
    ("s", 2, 768, 1024),     # a letterboxed 1024 x 768 image
    ("s", 1, 1024, 1024),
])
def test_records_match_generic_epilogue(size, B, H, W):
    th = _records(size, B, H, W)
    # the theta index is an integer bin; the calibrated model spreads it over the bins
    assert bool((th == th.round()).all()) and float(th.min()) >= 0 and float(th.max()) < 180
    assert th.unique().numel() > 20


def test_tta_records_match_generic_epilogue():
    m = _model("s")
    B, H, W = 2, 1024, 1024
    x = bench.synth_batch(B, 1).to(DEV).float() / 255
    outs = []
    for flags in (0, DETECT_GENERIC):
        plan = TTAPlan(m, B, H, W, DEV, compact_detect=True, conv_flags=flags)
        plan.pred.copy_(_sentinel(plan.pred.shape))
        pred = plan.forward(x)
        torch.cuda.synchronize()
        assert not torch.isnan(pred).any()
        outs.append(pred.clone())
        del plan
    _compare(outs[0], outs[1], "TTA records (de-scaled, flipped branches)")

