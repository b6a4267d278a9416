"""Exact checks of every conv, data-gradient and weight-gradient launch of the benchmarked plans, with integer operands.

When every operand is a small integer (exact in bf16) and the sum of |a*b| over each reduction stays below 2^24, every
product and every partial sum is exact in fp32 whatever the summation order, tile shape, split-K or atomic order.  A
kernel's fp32 result then equals the fp64 reference bit for bit, and its bf16 result equals that reference rounded once
to nearest-even: a dropped, duplicated, mis-swizzled or mis-addressed term changes the bits.  The fp32 accumulation of
wgmma is measured first (test_wgmma_accumulation_is_exact_below_2p24); the bound every case asserts, LIMIT, rests on it.

  * test_every_launch_matches_its_descriptor: each Conv / Wgrad object a plan owns, run alone on random integers, against
    tests/convref.py's evaluation of its own descriptor; inputs outside the read slice hold a large finite sentinel, the
    destination another sentinel, and every element outside the op's write mask must come back unchanged.
  * test_backward_composition_exact: the backward plan asks for the right operations (transposed / flipped weights, phase
    taps and offsets, accumulate vs overwrite, Detect's padded channel groups): every layer's dgrad launches equal
    conv2d_input of the forward weight and its wgrad conv2d_weight, bit for bit.
  * test_backward_stream_schedule: the full backward on real data, one stream, two streams and graph replay, agree.
"""
import math

import pytest
import torch

from tests.convref import conv_reference, expected, view_at, wgrad_reference
from tests.modelgen import build_mirror
from yolov5_obb_b200.conv import BIAS_HALVED, MODE_DETECT, Conv as ConvOp, Slice, WindowView
from yolov5_obb_b200.engine import InferenceEngine, TTAPlan
from yolov5_obb_b200.train_backward import BackwardPlan
from yolov5_obb_b200.train_engine import TrainArena, TrainEngine, _Carver
from yolov5_obb_b200.train_ops import Wgrad
from yolov5_obb_b200.train_step import freeze_layers

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LIMIT = 2 ** 24          # sums of |a*b| below this are exact in wgmma's fp32 accumulators (measured below)
IN_SENT = 4096.0         # input channels outside the read slice: finite (the pixel-pair view reads them against zero weights)
OUT_SENT = -12288.0      # destination elements the op must not write


def rint(shape, r):
    return torch.randint(-r, r + 1, tuple(shape), device=DEV).float()


def bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _compare(recs, before, what):
    """-> (bitwise?, worst error / tolerance ratio); asserts the write mask and everything outside it."""
    worst, exact = 0.0, True
    for rec in recs:
        after, m = rec.buf, rec.mask
        old = before[rec.buf.data_ptr()]
        moved = (bits(after) != bits(old)) & ~m
        assert not moved.any(), f"{what}: {int(moved.sum())} elements outside the write mask changed, first at " \
                                f"{moved.nonzero()[:4].tolist()}"
        if rec.tol is None:
            bad = bits(after) != bits(expected(rec))
            bad &= m
            assert not bad.any(), f"{what}: {int(bad.sum())} of {int(m.sum())} written elements differ, first at " \
                                  f"{bad.nonzero()[:4].tolist()}: got {after[bad][:4].tolist()}, " \
                                  f"want {expected(rec)[bad][:4].tolist()}"
            continue
        exact = False
        err = (after.double() - rec.value).abs()[m]
        tol = rec.tol[m]
        assert torch.equal(err[tol == 0], torch.zeros_like(err[tol == 0])), f"{what}: an exact element differs"
        assert torch.isfinite(err).all(), f"{what}: non-finite output"
        r = (err[tol > 0] / tol[tol > 0]).max().item() if (tol > 0).any() else 0.0
        assert r <= 1.0, f"{what}: error {r:.3f} x the epilogue bound"
        worst = max(worst, r)
    return exact, worst


def _real_rows(d, wp):
    if d.mode == MODE_DETECT:
        na = d.Cout // d.det_no
        bn = wp.shape[1] // na
        return torch.tensor([a * bn + j for a in range(na) for j in range(d.det_no)], device=DEV)
    return torch.arange(d.Cout, device=DEV)


def check_conv(op, st, what):
    d = op.desc
    x, wp, bp, out, res, out2x, det = op._keep
    detect = d.mode == MODE_DETECT
    dests = ([out.buf] if out is not None else []) + ([out2x.buf] if out2x is not None else []) + ([det["out"]] if det else [])
    for t in dests:
        t.fill_(OUT_SENT)
    if detect:      # small logits: the sigmoid is not saturated and the theta maxima tie often
        rx, rw, rb = 2, 1, 2
    elif d.act:     # SiLU's curved range
        rx, rw, rb = 2, 1, 4
    else:
        rx, rw, rb = 8, 8, 8
    if isinstance(x, WindowView):
        x.buf.copy_(rint(x.buf.shape, rx))
    else:
        if all(x.buf.data_ptr() != t.data_ptr() for t in dests):
            x.buf.fill_(IN_SENT)
        x.view().copy_(rint(x.view().shape, rx))
    rows = _real_rows(d, wp)
    real = torch.zeros(wp.shape[1:], dtype=torch.bool, device=DEV)
    real[rows, :d.Cin] = True
    assert not (wp[:, ~real] != 0).any(), f"{what}: packed weights are not zero outside the real region"
    wv = rint((wp.shape[0], len(rows), d.Cin), rw)
    if detect:
        wv *= torch.rand(wv.shape, device=DEV) < 4.0 / d.Cin
    wp[:, rows, :d.Cin] = wv.bfloat16()
    b = rint((len(rows),), rb)
    bp.zero_()
    bp[rows] = b * 0.5 if (d.flags & BIAS_HALVED) else b    # the buffer holds 0.5 * bias
    rr = 0
    if res is not None:
        rr = 8
        res.view().copy_(rint(res.view().shape, rr))
    bound = wp.shape[0] * d.Cin * rx * (wv.abs().max().item()) + rb + rr
    assert bound < LIMIT, (what, bound)
    recs = conv_reference(op)
    before = {t.data_ptr(): t.clone() for t in (r.buf for r in recs)}
    op.run()
    torch.cuda.synchronize()
    exact, worst = _compare(recs, before, what)
    st["conv"] += 1
    st["bitwise" if exact else "tolerance"] += 1
    st["worst"] = max(st["worst"], worst)
    if detect and d.det_decode == 2:
        st["ties"] += recs[0].ties
        st["rows"] += int(recs[0].mask.sum()) // recs[0].buf.shape[-1]


def check_wgrad(wg, st, what):
    d = wg.desc
    tensors = [t for t in wg._keep if isinstance(t, torch.Tensor)]

    def owner(ptr):
        c = [t for t in tensors if t.data_ptr() <= ptr < t.data_ptr() + t.numel() * t.element_size()]
        return max(c, key=lambda t: t.numel())

    npix = d.B * d.Ho * d.Wo
    r = max(1, min(8, math.isqrt((LIMIT // 2) // npix)))
    dzb, xb, dwb = owner(d.dz), owner(d.x), owner(d.dw)
    dzp = d.dz_pix_stride
    dzb.fill_(IN_SENT)
    dz = view_at(dzb, d.dz, (d.B, d.Ho, d.Wo, d.Cout), (dzp * d.Wo * d.Ho, dzp * d.Wo, dzp, 1))
    dz.copy_(rint(dz.shape, r))
    if d.x_row_stride:  # explicit strides (the stem's overlapping windows): the whole buffer is operand
        xb.copy_(rint(xb.shape, r))
    else:
        xb.fill_(IN_SENT)
        xp = d.x_pix_stride
        xv = view_at(xb, d.x, (d.B, d.Hi, d.Wi, d.Cin), (xp * d.Wi * d.Hi, xp * d.Wi, xp, 1))
        xv.copy_(rint(xv.shape, r))
    dwb.fill_(OUT_SENT)
    dw = wg._keep[0]
    dw.copy_(rint(dw.shape, 8))                    # accumulates onto what dW holds
    bound = npix * r * r + 8
    assert bound < LIMIT, (what, bound)
    recs = wgrad_reference(wg)
    before = {t.data_ptr(): t.clone() for t in (rr.buf for rr in recs)}
    wg.run()
    torch.cuda.synchronize()
    _compare(recs, before, what)
    st["wgrad"] += 1
    st["bitwise"] += 1


def _stats():
    return dict(conv=0, wgrad=0, bitwise=0, tolerance=0, worst=0.0, ties=0, rows=0)


# ---------------------------------------------------------------------------------------------------------------------
def test_wgmma_accumulation_is_exact_below_2p24():
    """One conv (Detect raw mode: fp32 out, one CTA sums all 4096 K terms of an element) and one wgrad (12 x 11 CTA tiles,
    so the split-K heuristic keeps one CTA per tile over all 8192 pixels) on non-negative integers whose sums reach 2^12,
    2^16, 2^20 and 2^23: the largest partial sum of each element is its final value, and every one must be exact."""
    torch.manual_seed(0)
    K, H, W, no = 4096, 32, 64, 64
    x = torch.empty(1, H, W, K, dtype=torch.bfloat16, device=DEV)
    wp = torch.zeros(1, no, K, dtype=torch.bfloat16, device=DEV)
    bp = torch.zeros(no + 32, device=DEV)
    out = torch.empty(1, H * W, no, device=DEV)
    det = dict(out=out, rows_per_image=H * W, row_off=0, no=no, decode=0, stride=1.0, anchors_px=[0.0] * 6)
    op = ConvOp(Slice.full(x), wp, bp, no, 1, 1, 0, False, det=det)
    Co, Ci, Ho, Wo = 1536, 2816, 64, 128
    dz = torch.empty(1, Ho, Wo, Co, dtype=torch.bfloat16, device=DEV)
    xw = torch.empty(1, Ho, Wo, Ci, dtype=torch.bfloat16, device=DEV)
    dw = torch.zeros(1, Co, Ci, device=DEV)
    wg = Wgrad(dz.data_ptr(), Co, xw.data_ptr(), Ci, dw, 1, Co, Ho, Wo, Ci, Ho, Wo, 1, 1, 0, keep=(dz, xw))
    for target in (2 ** 12, 2 ** 16, 2 ** 20, 2 ** 23):
        a = max(2, round(2 * math.sqrt(target / K)))
        x.copy_(torch.randint(0, a + 1, x.shape, device=DEV))
        wp.copy_(torch.randint(0, a + 1, wp.shape, device=DEV))
        rec = conv_reference(op)[0]
        out.zero_()
        op.run()
        torch.cuda.synchronize()
        top = rec.value.max().item()
        bad = int((bits(out) != bits(expected(rec))).sum())
        print(f"conv  max element {top:.0f} (2^{math.log2(top):.2f}): {bad} inexact")
        assert top < LIMIT and bad == 0
        a = max(2, round(2 * math.sqrt(target / (Ho * Wo))))
        dz.copy_(torch.randint(0, a + 1, dz.shape, device=DEV))
        xw.copy_(torch.randint(0, a + 1, xw.shape, device=DEV))
        dw.zero_()
        rec = wgrad_reference(wg)[0]
        wg.run()
        torch.cuda.synchronize()
        top = rec.value.max().item()
        bad = int((bits(dw) != bits(expected(rec).view(dw.shape))).sum())
        print(f"wgrad max element {top:.0f} (2^{math.log2(top):.2f}): {bad} inexact")
        assert top < LIMIT and bad == 0
        assert top >= target


# ---------------------------------------------------------------------------------------------------------------------
PLANS = [
    pytest.param("s", 16, 1024, 1024, "forward", id="yolov5s-b16-1024-forward"),
    pytest.param("s", 16, 1024, 1024, "records", id="yolov5s-b16-1024-records"),
    pytest.param("m", 16, 1024, 1024, "forward", id="yolov5m-b16-1024-forward"),
    pytest.param("m", 8, 1024, 1024, "train", id="yolov5m-b8-1024-train"),
    pytest.param("n", 2, 96, 160, "train", id="yolov5n-b2-96x160-train"),
    pytest.param("n", 2, 96, 160, "forward", id="yolov5n-b2-96x160-forward"),
    pytest.param("n", 2, 96, 160, "records", id="yolov5n-b2-96x160-records"),
]


class AliasCarver(_Carver):
    """A TrainEngine allocator for plans that are only read, never run: the buffers overlap in one shared allocation, so a
    plan's descriptors and schedules exist without its activations.  Buffer k starts 256 k bytes in (256-byte aligned as
    the arena carves them, and a start of its own: the plans tell buffers apart by their address); the offsets are counted
    as the arena counts them, and channel slices keep their offsets within their buffer.  Nothing may run on such a plan."""

    def __init__(self, device):
        super().__init__(None, device)
        self.buf = torch.empty(0, dtype=torch.uint8, device=device)
        self.n = 0

    def take(self, shape, dtype):
        n = math.prod(int(s) for s in shape) * torch.empty((), dtype=dtype).element_size()
        a = TrainArena.ALIGN
        self.off = (self.off + a - 1) // a * a + n
        start = self.n * a
        self.n += 1
        if start + n > self.buf.numel():   # (views of the old allocation keep it alive)
            self.buf = torch.empty(max(start + n, 2 * self.buf.numel()) + 1024 * a, dtype=torch.uint8, device=self.device)
        return self.buf[start:start + n].view(dtype).view(tuple(shape))


def plan_launches(size, B, H, W, kind, freeze=None, key_only=False):
    """(conv ops, wgrad ops, what keeps them alive) of the yolov5{size} plan of `kind` at B x H x W, each built by the code
    path its entry point uses: every launch the plan makes, in plan order.
      forward / records   InferenceEngine (Model.forward; detect_records, SceneDetector, run_images);
      tta / tta-records   the three InferenceEngines of TTAPlan (forward_augment; detect_records(augment=True));
      train               TrainEngine's forward convs and Detect convs, then the dgrads of the BackwardPlan that
                          TrainEngine.backward builds for the requires_grad flags train.py --freeze `freeze` leaves
                          (None: every parameter trains).  A multi-scale size is a train plan of that size.
    key_only: a train plan's buffers all alias one allocation (AliasCarver): its launches can be read but not run."""
    m = build_mirror(size, nc=15, seed=0)
    wgrads = []
    if kind == "train":
        m = m.train().to(DEV)
        if freeze is not None:
            freeze_layers(m, [freeze] if isinstance(freeze, int) else list(freeze))
        eng = TrainEngine(m, B, H, W, DEV, carver=AliasCarver(torch.device(DEV)) if key_only else None)
        plan = BackwardPlan(eng, tuple(p.requires_grad for p in m.parameters()))
        convs = [lay.conv for lay in eng.conv_layers] + list(eng.det_convs)
        bwd = []
        for part in plan.det_parts + plan.conv_parts:
            bwd += part.get("dgrad_ops", [])
            if "wgrad" in part:
                wgrads.append(part["wgrad"])
        # the parts list every conv / wgrad object the backward plan keeps
        assert {id(o) for o in plan.keep if isinstance(o, (ConvOp, Wgrad))} == {id(o) for o in bwd + wgrads}
        s2 = [len(p["dgrad_ops"]) for p in plan.conv_parts if "dgrad_ops" in p and p["lay"].mod.conv.stride[0] == 2]
        assert s2 and all(n == 4 for n in s2), s2
        if freeze is None:
            assert len(wgrads) == len(plan.det_parts) + len(plan.conv_parts)
        return convs + bwd, wgrads, (m, eng, plan)
    assert freeze is None and not key_only
    if kind in ("tta", "tta-records"):
        tta = TTAPlan(m, B, H, W, DEV, compact_detect=kind == "tta-records")
        return [op for e in tta.engines for op in e.convs], wgrads, (m, tta)
    assert kind in ("forward", "records"), kind
    eng = InferenceEngine(m, B, H, W, DEV, compact_detect=kind == "records")
    return list(eng.convs), wgrads, (m, eng)


@pytest.mark.parametrize("size,B,H,W,kind", PLANS)
def test_every_launch_matches_its_descriptor(size, B, H, W, kind, freeze=None):
    """Every launch against its own descriptor (tests/convref.py).  Bitwise: every act=False conv (train forward, every dgrad
    form), raw Detect rows, every wgrad (split-K over the whole pixel axis, the stem's window view, Detect's padded
    channel groups), out2x against the repeated output.  Theta index of records: the first maximum, exactly.  Within a bound
    of the epilogue's own approximation, on an exact pre-activation:
      * SiLU convs: tanh.approx's relative error (2^-11 documented, 2^-10 used) times |h| |tanh h|, h = (acc + bias) / 2,
        plus the fma's fp32 rounding, then one bf16 rounding of the result (2^-8 |y|); a residual is added in fp32 and the
        sum rounded once (DESIGN §7), so it adds an fp32 rounding and no second bf16 one;
      * decoded Detect rows and records: the sigmoid 0.5 tanh.approx(0.5 x) + 0.5 errs by at most half of tanh's error (+ one
        fp32 rounding), propagated through the decode (x 2 stride for xy, x 8 anchor for wh) plus the fp32 roundings of the
        decode arithmetic."""
    torch.manual_seed(2)
    convs, wgrads, _ = plan_launches(size, B, H, W, kind, freeze)
    st = _stats()
    for i, op in enumerate(convs):
        check_conv(op, st, f"conv {i}")
    for i, wg in enumerate(wgrads):
        check_wgrad(wg, st, f"wgrad {i}")
    print(f"\n{size} b{B} {H}x{W} {kind}: {st['conv']} conv and {st['wgrad']} wgrad "
          f"launches checked; {st['bitwise']} bitwise, {st['tolerance']} within the epilogue bound "
          f"(worst {st['worst']:.3f} of it)" + (f"; theta ties in {st['ties']} of {st['rows']} records rows"
                                                   if kind.endswith("records") else ""))
    assert st["conv"] == len(convs) and st["wgrad"] == len(wgrads)
    if kind.endswith("records"):
        assert st["ties"] > 0


# ---------------------------------------------------------------------------------------------------------------------
def _nchw(t):
    return t.permute(0, 3, 1, 2).double()


def _s2d_from_image(xs, img):
    """x_s2d[b, i, 1 + j, (dy*2+dx)*3 + c] = img[b, c, 2i+dy, 2j+dx]; pad pixels and channels 12-15 zero."""
    xs.zero_()
    for dy in range(2):
        for dx in range(2):
            xs[:, :, 1:-1, (dy * 2 + dx) * 3:(dy * 2 + dx) * 3 + 3] = img[:, :, dy::2, dx::2].permute(0, 2, 3, 1).bfloat16()


def _wgrad_fp64(x, shape, dz, s, p):
    g = torch.zeros(shape, dtype=torch.float64, device=DEV)
    for b in range(x.shape[0]):  # per image; integer partial sums add exactly in fp64
        g += torch.nn.grad.conv2d_weight(x[b:b + 1], shape, dz[b:b + 1], stride=s, padding=p).round()
    return g


def _check_flat(plan, dwv, want, snap, what):
    m = torch.zeros(plan.flat.shape, dtype=torch.bool, device=DEV)
    off = (dwv.data_ptr() - plan.flat.data_ptr()) // 4
    m[off:off + dwv.numel()] = True
    assert torch.equal(bits(plan.flat[~m]), bits(snap[~m])), f"{what}: wgrad wrote outside its parameter"
    bad = bits(dwv.reshape(-1)) != bits(want.reshape(-1).float())
    assert not bad.any(), f"{what}: {int(bad.sum())} of {dwv.numel()} weight-gradient elements differ"


def test_backward_composition_exact():
    """yolov5m, b8, 1024x1024 (the benchmarked train step): backward_composition."""
    backward_composition("m", 8, 1024, 1024)


def backward_composition(size, B, H, W):
    """The yolov5{size} B x H x W train plan with integer weights: every layer's dgrad launches, run on integer dz, equal
    conv2d_input of the FORWARD weight with the layer's stride and padding (onto the integers gx held when the plan
    accumulates there, over a sentinel when it overwrites); each stride-2 phase changes only pixels of its parity; every
    wgrad equals conv2d_weight (the stem's in the space-to-depth layout, Detect's without the padding channels of its dz).
    Bitwise.  Returns (dgrad layers, accumulating ones, wgrad layers)."""
    torch.manual_seed(3)
    m = build_mirror(size, nc=15, seed=0).train().to(DEV)
    eng = TrainEngine(m, B, H, W, DEV)
    plan = BackwardPlan(eng)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.Conv2d):
                mod.weight.copy_(rint(mod.weight.shape, 3))
                if mod.bias is not None:
                    mod.bias.copy_(rint(mod.bias.shape, 3))
    plan.refresh()
    det = m.model[-1]
    n_dgrad = n_wgrad = n_acc = 0

    def dgrad(part, want_fn, what):
        nonlocal n_dgrad, n_acc
        ops = part["dgrad_ops"]
        gx = ops[0]._keep[3]
        acc = bool(ops[0].desc.res)
        assert all(bool(o.desc.res) == acc for o in ops)
        gx.buf.fill_(OUT_SENT)
        if acc:
            gx.view().copy_(rint(gx.view().shape, 8))
            n_acc += 1
        g0 = _nchw(gx.view()) if acc else 0
        snap = gx.buf.clone()
        prev = snap
        for i, op in enumerate(ops):
            op.run()
            torch.cuda.synchronize()
            if len(ops) == 4:  # phase (ph, pw) = divmod(i, 2) writes pixels (2i+ph, 2j+pw) only
                ph, pw = divmod(part["dgrad_s2"][i][0], 2)
                moved = (bits(gx.buf) != bits(prev)).any(-1)
                par = torch.zeros(moved.shape[1:], dtype=torch.bool, device=DEV)
                par[ph::2, pw::2] = True
                assert not (moved & ~par).any(), f"{what}: phase {ph}{pw} wrote pixels of another parity"
                prev = gx.buf.clone()
        outside = torch.ones(gx.buf.shape[-1], dtype=torch.bool, device=DEV)
        outside[gx.c_off:gx.c_off + gx.C] = False
        assert torch.equal(bits(gx.buf[..., outside]), bits(snap[..., outside])), f"{what}: dgrad wrote outside gx"
        want = (want_fn() + g0).permute(0, 2, 3, 1)
        assert want.abs().max().item() < LIMIT
        bad = bits(gx.view()) != bits(want.float().bfloat16())
        assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.numel()} input-gradient elements differ"
        n_dgrad += 1

    for part in plan.conv_parts:
        lay = part["lay"]
        conv = lay.mod.conv
        k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        what = f"{type(lay.mod).__name__} {conv.in_channels}->{conv.out_channels} k{k} s{s} at {lay.z.H}x{lay.z.W}"
        dz = part["dz"]
        dz.copy_(rint(dz.shape, 2))
        dzn = _nchw(dz)
        wf = conv.weight.detach().double()
        plan.flat.fill_(OUT_SENT)
        if lay.stem:
            img = rint((B, 3, H, W), 2)
            _s2d_from_image(eng.x_s2d, img)
            dwv = part["stem_dw"]
            dwv.copy_(rint(dwv.shape, 8))
            w0 = dwv.double().view(3, conv.out_channels, 3, 16)       # [ty][co][tx][ch16]
            g = _wgrad_fp64(img.double(), wf.shape, dzn, 2, 2)         # [co, c, 6, 6]
            want = w0.clone()
            for dy in range(2):
                for dx in range(2):
                    for c in range(3):   # w[co, c, 2ty+dy, 2tx+dx] -> dw[ty][co][tx][(dy*2+dx)*3 + c]
                        want[:, :, :, (dy * 2 + dx) * 3 + c] += g[:, c, dy::2, dx::2].permute(1, 0, 2)
            snap = plan.flat.clone()
            part["wgrad"].run()
            torch.cuda.synchronize()
            assert torch.equal(bits(plan.flat), bits(snap)), f"{what}: stem wgrad wrote into the flat gradient"
            bad = bits(dwv) != bits(want.reshape(-1).float())
            assert not bad.any(), f"{what}: {int(bad.sum())} stem weight-gradient elements differ"
            n_wgrad += 1
            continue
        x = lay.x
        x.buf.fill_(IN_SENT)
        x.view().copy_(rint(x.view().shape, 2))
        xn = _nchw(x.view())
        dwv = plan.pgrad[conv.weight]
        dwv.copy_(rint(dwv.shape, 8))
        want = dwv.double() + _wgrad_fp64(xn, wf.shape, dzn, s, p)
        assert want.abs().max().item() < LIMIT
        snap = plan.flat.clone()
        part["wgrad"].run()
        torch.cuda.synchronize()
        _check_flat(plan, dwv, want, snap, what)
        n_wgrad += 1
        dgrad(part, lambda: torch.nn.grad.conv2d_input(xn.shape, wf, dzn, stride=s, padding=p).round(), what)

    for part in plan.det_parts:
        mi, bn, dzd = part["mi"], part["bn"], part["dzd"]
        what = f"Detect level {part['l']}"
        x = eng.det_convs[part["l"]]._keep[0]
        dzd.copy_(rint(dzd.shape, 2))            # the padding channels of every anchor group too: they must be skipped
        real = dzd.view(*dzd.shape[:3], det.na, bn)[..., :det.no].reshape(-1, det.na * det.no).double()
        x.buf.fill_(IN_SENT)
        x.view().copy_(rint(x.view().shape, 2))
        xf = x.view().reshape(-1, x.C).double()
        wf = mi.weight.detach().double()[:, :, 0, 0]
        plan.flat.fill_(OUT_SENT)
        dwv = plan.pgrad[mi.weight]
        dwv.copy_(rint(dwv.shape, 8))
        want = dwv.double() + (real.t() @ xf).view(dwv.shape)
        snap = plan.flat.clone()
        part["wgrad"].run()
        torch.cuda.synchronize()
        _check_flat(plan, dwv, want, snap, what)
        n_wgrad += 1
        shp = x.view().shape
        dgrad(part, lambda: (real @ wf).view(shp[0], shp[1], shp[2], x.C).permute(0, 3, 1, 2), what)
    print(f"\nyolov5{size} b{B} {H}x{W} backward composition: {n_dgrad} dgrad layers ({n_acc} accumulating) and {n_wgrad} "
          f"wgrad layers bitwise")
    assert n_wgrad == len(plan.conv_parts) + len(plan.det_parts)
    return n_dgrad, n_acc, n_wgrad


def test_backward_stream_schedule(monkeypatch):
    """The full backward of the yolov5m b8 1024x1024 train plan on real data, three ways: one stream (Y5OBB_WGRAD_STREAM=0),
    the default two-stream first call, and its graph replay.  wgrad's fp32 atomics and the max-pool backward's atomics
    reorder sums, so the gradients agree to a relative L2 error of 1e-3 per buffer; a missing cross-stream dependency would
    read a stale or half-written operand and show as an O(1) difference."""
    torch.manual_seed(4)
    B, H, W = 8, 1024, 1024
    m = build_mirror("m", nc=15, seed=0).train().to(DEV)
    eng = TrainEngine(m, B, H, W, DEV)
    g = torch.Generator().manual_seed(5)
    x = torch.rand(B, 3, H, W, generator=g).to(DEV)
    with torch.no_grad():
        outs = eng.forward(x)
    G = [(torch.randn(o.shape, generator=g) * 0.05).to(DEV) for o in outs]
    monkeypatch.setenv("Y5OBB_WGRAD_STREAM", "0")
    one = BackwardPlan(eng)
    monkeypatch.delenv("Y5OBB_WGRAD_STREAM")
    two = BackwardPlan(eng)
    assert one.side is None and two.side is not None

    def grads(plan):
        plan.run(G)
        torch.cuda.synchronize()
        return [t.clone() for t in plan.gbuf.values()] + [plan.flat.clone()]

    ref = grads(one)
    runs = {"two streams": grads(two)}
    runs["graph replay"] = grads(two)
    assert two._graph is not None
    names = [f"gradient buffer {i}" for i in range(len(ref) - 1)] + ["flat parameter gradient"]
    for label, got in runs.items():
        worst, equal = 0.0, 0
        for n, a, b in zip(names, ref, got):
            if torch.equal(bits(a), bits(b)):
                equal += 1
                continue
            rel = ((a.float() - b.float()).norm() / a.float().norm().clamp_min(1e-30)).item()
            assert rel < 1e-3, (label, n, rel)
            worst = max(worst, rel)
        print(f"\nbackward, {label} vs one stream: {equal} of {len(ref)} buffers bitwise equal, worst relative L2 of the "
              f"others {worst:.2e}")
