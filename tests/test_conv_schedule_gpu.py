"""The conv kernel's launch schedule changes where a tile runs, never what it computes.

For every conv launch of the yolov5s b16 1024x1024 records plan (the benchmark's inference) and of the yolov5m b8 1024x1024
train plan (forward convs and every dgrad launch), the default plan and a twin created from the same descriptor with
Y5OBB_CONV_ONE_CTA (one CTA per SM everywhere) run on the same random operands: every destination buffer, sentinels
outside the write region included, must come back bit-identical.

The schedule is checked per launch: an N tile of more than 96 instruction columns runs one CTA per SM; a narrower one runs
two, unless it is a row-shift layer (the summation order the full-SM plan fixes) whose row-shift ring does not fit half of
the shared memory - one load per tap always fits there.  For the records plan the launches are also named: convs 0-5, 8,
10 and 36 (the stem, layer 1, the C3 blocks of layers 2 and 4, the top-down C3 at 128^2) two, the 3x3 64 -> 64 Bottleneck
convs 9, 11 and 37 one.
"""
import ctypes

import pytest
import torch

from tests.modelgen import build_mirror
from yolov5_obb_b200 import _lib
from yolov5_obb_b200.conv import ONE_CTA, ConvDesc
from yolov5_obb_b200.engine import InferenceEngine
from yolov5_obb_b200.train_backward import BackwardPlan
from yolov5_obb_b200.train_engine import TrainEngine

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENT = -12288.0


def instr_n(bn):
    return 16 if bn <= 16 else (bn + 31) // 32 * 32


class Twin:
    """The same descriptor with extra flags, created through the C ABI."""

    def __init__(self, op, flags):
        self.desc = ConvDesc.from_buffer_copy(op.desc)
        self.desc.flags |= flags
        self._h = ctypes.c_void_p()
        rc = _lib.lib().y5obb_conv_create(ctypes.byref(self.desc), ctypes.byref(self._h))
        _lib.check(rc, "y5obb_conv_create")
        self.device = op.device

    def run(self):
        _lib.check(_lib.lib().y5obb_conv_run(self._h, _lib.stream_ptr(self.device)), "y5obb_conv_run")

    def schedule(self):
        cta = ctypes.c_int()
        _lib.check(_lib.lib().y5obb_conv_schedule(self._h, ctypes.byref(cta), None, None, None), "y5obb_conv_schedule")
        return cta.value

    def close(self):
        _lib.lib().y5obb_conv_destroy(self._h)


def _buffers(op):
    x, wp, bp, out, res, out2x, det = op._keep
    dests = [s.buf for s in (out, out2x) if s is not None] + ([det["out"]] if det else [])
    srcs = [x.buf] + ([res.buf] if res is not None else [])
    return srcs, dests


def check_same(op, what, counts):
    srcs, dests = _buffers(op)
    g = torch.Generator(device=DEV).manual_seed(counts["n"])
    for t in dests:
        t.fill_(SENT)
    for t in srcs:   # after the sentinels: an input or a residual may share the destination's buffer
        t.copy_(torch.randn(t.shape, generator=g, device=DEV).to(t.dtype))
    every = list({t.data_ptr(): t for t in srcs + dests}.values())
    snap = [t.clone() for t in every]
    before = [t.clone() for t in dests]
    op.run()
    torch.cuda.synchronize()
    got = [t.clone() for t in dests]
    for t, s in zip(every, snap):
        t.copy_(s)
    twin = Twin(op, ONE_CTA)
    try:
        assert twin.schedule() == 1, what
        twin.run()
        torch.cuda.synchronize()
    finally:
        twin.close()
    for a, b, old in zip(got, dests, before):
        bits = (lambda t: t.view(torch.int16)) if a.element_size() == 2 else (lambda t: t.view(torch.int32))
        bad = bits(a) != bits(b)
        assert not bad.any(), f"{what}: {int(bad.sum())} elements differ between the default and the one-CTA plan"
        assert (bits(b) != bits(old)).any(), f"{what}: nothing written"
    info = op.info()
    ni = instr_n(info["block_n"])
    if ni > 96:
        assert info["ctas_per_sm"] == 1, (what, ni, info)
    else:
        assert info["ctas_per_sm"] == 2 or info["rowshift"] == 1, (what, ni, info)
    counts["ni96"] += ni <= 96
    counts["n"] += 1
    counts["two"] += info["ctas_per_sm"] == 2
    return info["ctas_per_sm"]


@pytest.mark.parametrize("size,B,kind", [("s", 16, "records"), ("m", 8, "train")], ids=["yolov5s-b16-records", "yolov5m-b8-train"])
def test_schedule_is_bit_identical_to_one_cta(size, B, kind):
    torch.manual_seed(0)
    m = build_mirror(size, nc=15, seed=0)
    if kind == "train":
        m = m.train().to(DEV)
        eng = TrainEngine(m, B, 1024, 1024, DEV)
        plan = BackwardPlan(eng)
        convs = [lay.conv for lay in eng.conv_layers] + list(eng.det_convs)
        for part in plan.det_parts + plan.conv_parts:
            convs += part.get("dgrad_ops", [])
    else:
        eng = InferenceEngine(m.to(DEV), B, 1024, 1024, DEV, compact_detect=True)
        convs = list(eng.convs)
    counts = dict(n=0, two=0, ni96=0)
    ctas = [check_same(op, f"conv {i}", counts) for i, op in enumerate(convs)]
    if kind == "records":
        assert [i for i, c in enumerate(ctas) if c == 2] == [0, 1, 2, 3, 4, 5, 8, 10, 36], ctas
        assert all(instr_n(convs[i].info()["block_n"]) <= 96 and ctas[i] == 1 for i in (9, 11, 37)), ctas
    print(f"\n{size} b{B} {kind}: {counts['n']} launches bit-identical to one CTA per SM; {counts['two']} of the "
          f"{counts['ni96']} with N tiles <= 96 ran two per SM")
    assert counts["n"] == len(convs) and counts["two"] > 0
