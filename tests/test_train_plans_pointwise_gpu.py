"""Element-by-element checks of the training kernels between the convolutions (csrc/bn_train.cu) against fp64
(tests/bnref.py): batch statistics and the running-stat update, normalise + SiLU into a channel slice (residual, 2x
up-sampled copy), the BatchNorm / SiLU backward (dz, dgamma, dbeta, residual pass-through) and the gradient-routing kernels.

Bit-exact where the arithmetic is order-free or restatable in torch (the routing kernels, the max-pool backward on dyadic
gradients, the residual pass-through, dgamma / dbeta from the kernel's own sums, mean and scale from its own sums, the
2x copies); elsewhere each element is held to a bound derived from the kernel's fp32 arithmetic (bnref's docstring).  Every
destination lives in a wider buffer (pix_stride > C, c_off != 0) filled with a sentinel that must come back unchanged
outside the op's write mask, and the reduction scratch is filled with NaN before every launch.

  1. each kernel through the C ABI at shapes chosen for its launch geometry (idle threads, lanes < 16, the second
     column group at C > 2048, chunks that do not divide npix) and |mean| / sigma in {0, 10, 100, 300} (the statistics'
     quality bar is asserted up to 10; 100 and 300 are printed);
  2. every BatchNorm forward launch of the yolov5m b8 1024x1024 train plan (bench.py's train leg) and of a small yolov5s
     plan with the arguments TrainEngine._forward_eager passes, and every non-conv step of their BackwardPlan alone through
     its own closure;
  3. the accumulate flags of the backward plan: each layer output's gradient range gets one overwrite, then one accumulate
     per further consumer, counted from the model graph (a layer whose gradient a frozen backbone prunes gets none).
Section 2's checks take any train plan: a frozen backbone (train.py --freeze) and a plan carved from a multi-scale run's
arena; tests/test_train_plans_pointwise_wide_gpu.py runs them on the P6, multi-scale and frozen plans.
Worst error-to-bound ratios per launch kind are printed at the end of the module (run with -s)."""
import inspect
import time

import pytest
import torch

from tests import bnref
from tests.bnref import U, gamma, stat_chain, ulp32
from tests.modelgen import build_mirror
from yolov5_obb_b200 import _lib
from yolov5_obb_b200.layout import _is, grad_liveness, shapes, sources
from yolov5_obb_b200.train_backward import BackwardPlan
from yolov5_obb_b200.train_engine import TrainEngine, _PoolLayer
from yolov5_obb_b200.train_step import freeze_layers

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
IN_SENT = 4096.0        # input channels outside the read slice
OUT_SENT = -12288.0     # destination elements the op must not write
EPS, MOM = 1e-3, 0.03
CHUNK_ELEMS = 1 << 25   # fp64 references are formed this many elements (256 MB) at a time

WORST = {}
LIMIT_RATIO = []


def note(kind, r):
    WORST[kind] = max(WORST.get(kind, 0.0), float(r))
    assert r <= 1.0, f"{kind}: error {r:.3f} x its bound"


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    print(f"\n[pointwise] worst error / bound per launch kind ({time.time() - t0:.0f} s for the module):")
    for k in sorted(WORST):
        print(f"  {k:28s} {WORST[k]:.3e}")
    for line in LIMIT_RATIO:
        print(f"  statistics beyond the asserted range: {line}")


def lib():
    return _lib.lib()


def stream():
    return _lib.stream_ptr(torch.device(DEV))


def sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def slab(lead, C, extra=16, c_off=8, fill=OUT_SENT, dtype=torch.bfloat16):
    """A [*lead, C + extra] buffer filled with `fill` and its channel slice [c_off, c_off + C) (16-byte aligned)."""
    buf = torch.full(tuple(lead) + (C + extra,), fill, dtype=dtype, device=DEV)
    return buf, buf[..., c_off:c_off + C]


def f32(C, fill=float("nan")):
    return torch.full((C,), fill, dtype=torch.float32, device=DEV)


def scratch(C):
    return torch.full((int(lib().y5obb_bn_scratch_floats(C)),), float("nan"), dtype=torch.float32, device=DEV)


def unchanged(buf, before, mask, what):
    """Every element of `buf` outside `mask` (bool, broadcastable) equals `before` bit for bit."""
    moved = (bits(buf) != bits(before)) & ~mask
    assert not moved.any(), f"{what}: {int(moved.sum())} elements outside the write mask changed, first at " \
                            f"{moved.nonzero()[:4].tolist()}"


def chan_mask(buf, c_off, C):
    m = torch.zeros(buf.shape[-1], dtype=torch.bool, device=DEV)
    m[c_off:c_off + C] = True
    return m


def channel_blocks(npix, C):
    w = max(8, min(C, CHUNK_ELEMS // max(1, npix)))
    return [(c0, min(C, c0 + w)) for c0 in range(0, C, w)]


def gen_z(shape, C, ratio, g):
    """bf16 data with per-channel sigma in [0.5, 2) and |mean| = ratio * sigma (random sign)."""
    sig = 0.5 + 1.5 * torch.rand(C, device=DEV, generator=g)
    mu = ratio * sig * torch.sign(torch.rand(C, device=DEV, generator=g) - 0.5)
    return (torch.randn(tuple(shape) + (C,), device=DEV, generator=g) * sig + mu).bfloat16()


def rand_bn(C, g):
    return dict(gamma=(0.5 + torch.rand(C, device=DEV, generator=g)), beta=0.3 * torch.randn(C, device=DEV, generator=g),
                rm=torch.randn(C, device=DEV, generator=g), rv=0.5 + torch.rand(C, device=DEV, generator=g))


# =========================================================================================================== references
def check_sums(zv, npix, C, s, q, kind):
    """sum / sumsq of y5obb_bn_stats against fp64 sums of the same bf16 values, within gamma(d) * sum|term|."""
    z2 = zv.reshape(npix, C)
    d = stat_chain(npix, C, sms())
    worst = 0.0
    for c0, c1 in channel_blocks(npix, C):
        x = z2[:, c0:c1].double()
        es = (s[c0:c1].double() - x.sum(0)).abs() / (gamma(d) * x.abs().sum(0)).clamp(min=1e-300)
        eq = (q[c0:c1].double() - (x * x).sum(0)).abs() / (gamma(d) * (x * x).sum(0)).clamp(min=1e-300)
        worst = max(worst, es.max().item(), eq.max().item())
    note(kind, worst)


def check_batch_stats(zv, npix, C, s, q, bn, out, ratio, kind):
    """mean / invstd / scale / shift / running statistics of y5obb_bn_batch_stats.  s, q: the same launch geometry's fp32
    sums (y5obb_bn_stats, which y5obb_bn_batch_stats forms in the same order); out: dict(scale, shift, mean, invstd, rm, rv)
    written by the kernel; bn: its inputs.  From the kernel's own sums: mean = (float)(sum / n) bit for bit, invstd within
    one fp32 ulp of fp64, scale = RN(gamma * invstd) bit for bit, shift within one ulp of beta - mean * scale (either
    contraction), running statistics by torch's rule (unbiased variance).  Then against the exact statistics of the bf16
    input: mean within the summation bound, and invstd within 2^-10 relative up to |mean| / sigma = 10.  Beyond that the
    fp32 E[z^2] - E[z]^2 loses the variance to cancellation (DESIGN.md section 7): 100 and 300 are printed, not asserted."""
    n = npix
    m64, var64, iv64 = bnref.finalize_ref(s, q, n, EPS)
    assert torch.equal(bits(out["mean"]), bits(m64.float())), f"{kind}: mean is not (float)(sum / n) of its own sums"
    note(f"{kind} invstd (ulp)", ((out["invstd"].double() - iv64).abs() / ulp32(iv64)).max().item())
    assert torch.equal(bits(out["scale"]), bits((bn["gamma"].double() * out["invstd"].double()).float())), \
        f"{kind}: scale != RN(gamma * invstd)"
    fused = bn["beta"].double() - out["mean"].double() * out["scale"].double()
    ok = ((out["shift"].double() - fused).abs() <= ulp32(fused)) | \
        torch.eq(bits(out["shift"]), bits(bn["beta"] - (out["mean"] * out["scale"])))
    assert ok.all(), f"{kind}: shift differs from beta - mean * scale by more than one ulp"
    mom1 = float(torch.tensor(1.0 - MOM, dtype=torch.float32))   # (1.0f - momentum)
    momf = float(torch.tensor(MOM, dtype=torch.float32))
    unb = var64 * n / (n - 1.0) if n > 1 else var64
    for key, new, old in (("rm", out["mean"].double(), bn["rm"]), ("rv", unb, bn["rv"])):
        want = mom1 * old.double() + momf * new
        tol = 4 * U * (mom1 * old.double().abs() + momf * new.abs()) + ulp32(want)
        note(f"{kind} running stats", ((out[key].double() - want).abs() / tol).max().item())
    z2 = zv.reshape(npix, C)
    d = stat_chain(npix, C, sms())
    epsd = float(torch.tensor(EPS, dtype=torch.float32))
    for c0, c1 in channel_blocks(npix, C):
        x = z2[:, c0:c1].double()
        mt = x.mean(0)
        ivt = 1.0 / torch.sqrt(((x - mt) ** 2).mean(0) + epsd)
        mtol = gamma(d) * x.abs().sum(0) / n + ulp32(mt)
        note(f"{kind} mean", ((out["mean"][c0:c1].double() - mt).abs() / mtol).max().item())
        rel = ((out["invstd"][c0:c1].double() - ivt).abs() / ivt).max().item()
        if ratio > 10:
            LIMIT_RATIO.append(f"{kind} npix {npix} C {C} |mean|/sigma {ratio}: invstd relative error {rel:.2e} "
                               f"(2^-10 = {2 ** -10:.2e})")
        else:
            note(f"{kind} invstd quality", rel / 2 ** -10)


def check_apply(zv, scale, shift, act, resv, y, ybuf, y_before, y_coff, y2x, kind):
    """y (a slice of ybuf at channel y_coff) against bnref.apply_ref; y2x = (buffer, before, c_off) or None: its four
    copies of every pixel equal y bit for bit and nothing else in it moves."""
    B, H, W, C = zv.shape
    npix = B * H * W
    z2, y2 = zv.reshape(npix, C), y.reshape(npix, C)
    r2 = resv.reshape(npix, C) if resv is not None else None
    worst = 0.0
    for c0, c1 in channel_blocks(npix, C):
        want, tol = bnref.apply_ref(z2[:, c0:c1], scale[c0:c1], shift[c0:c1], act, r2[:, c0:c1] if r2 is not None else None)
        err = (y2[:, c0:c1].double() - want).abs()
        assert torch.isfinite(err).all(), f"{kind}: non-finite output"
        worst = max(worst, (err / tol).max().item())
    note(kind, worst)
    unchanged(ybuf, y_before, chan_mask(ybuf, y_coff, C), f"{kind} y")
    if y2x is not None:
        ubuf, u_before, u_coff = y2x
        u = ubuf[..., u_coff:u_coff + C]
        for dh in range(2):
            for dw in range(2):
                assert torch.equal(bits(u[:, dh::2, dw::2]), bits(y)), f"{kind}: y2x quadrant ({dh}, {dw}) != y"
        unchanged(ubuf, u_before, chan_mask(ubuf, u_coff, C), f"{kind} y2x")


def check_bwd(zv, dyv, st, act, s1, s2, dz, gres, dgb, kind):
    """y5obb_bn_silu_bwd's outputs.  st: dict(scale, shift, mean, invstd) the launch read; s1 / s2: its sum_du / sum_dux;
    dz: [..., C] (its own buffer, fully written); gres: None or (slice after, old slice, accumulate?);
    dgb: (dgamma, dbeta, old dgamma, old dbeta, param_accumulate?)."""
    C = zv.shape[-1]
    npix = zv.numel() // C
    z2, d2, dz2 = zv.reshape(npix, C), dyv.reshape(npix, C), dz.reshape(npix, C)
    d = stat_chain(npix, C, sms())
    ws = wq = wz = 0.0
    for c0, c1 in channel_blocks(npix, C):
        sl = slice(c0, c1)
        z = z2[:, sl].double()
        du, e_du = bnref.du_ref(z2[:, sl], d2[:, sl], st["scale"][sl], st["shift"][sl], act)
        m, iv = st["mean"][sl].double(), st["invstd"][sl].double()
        bound_s = gamma(d) * du.abs().sum(0) + e_du.sum(0)
        ws = max(ws, ((s1[sl].double() - du.sum(0)).abs() / (1.001 * bound_s).clamp(min=1e-300)).max().item())
        want_q = iv * (du * (z - m)).sum(0)
        bound_q = gamma(d + 3) * iv * ((du * z).abs().sum(0) + m.abs() * du.abs().sum(0)) + \
            iv * (e_du * (z - m).abs()).sum(0)
        wq = max(wq, ((s2[sl].double() - want_q).abs() / (1.001 * bound_q).clamp(min=1e-300)).max().item())
        want, tol = bnref.dz_ref(z2[:, sl], du, e_du, st["scale"][sl], st["mean"][sl], st["invstd"][sl], s1[sl], s2[sl], npix)
        err = (dz2[:, sl].double() - want).abs()
        assert torch.isfinite(err).all(), f"{kind}: non-finite dz"
        wz = max(wz, (err / tol).max().item())
    note(f"{kind} sum_du", ws)
    note(f"{kind} sum_dux", wq)
    note(f"{kind} dz", wz)
    if gres is not None:
        g, old, acc = gres
        want = (old.float() + dyv.float()).bfloat16() if acc else dyv
        assert torch.equal(bits(g), bits(want)), f"{kind}: residual gradient is not {'RN(old + dy)' if acc else 'dy'}"
    if dgb is not None:
        dg, db, odg, odb, pacc = dgb
        assert torch.equal(bits(dg), bits((odg if pacc else torch.zeros_like(odg)) + s2)), f"{kind}: dgamma"
        assert torch.equal(bits(db), bits((odb if pacc else torch.zeros_like(odb)) + s1)), f"{kind}: dbeta"


# =========================================================================================================== 1. kernels
STAT_C = [8, 16, 48, 96, 384, 768, 1280, 2056]


def stat_npix(C, which):
    lanes = bnref.stat_layout(C)[2]
    full = lanes * 16 * 4 * sms()          # the last npix at which every block still gets >= 16 pixels per lane
    return {"2": 2, "lanes-1": lanes - 1, "full-1": full - 1, "full+1": full + 1}[which]


def run_stats(zv, stride, npix, C, bn):
    """y5obb_bn_stats then y5obb_bn_batch_stats on the same slice (NaN scratch before each) -> (s, q, out)."""
    L, st = lib(), stream()
    s, q = f32(C), f32(C)
    scr = scratch(C)
    assert L.y5obb_bn_stats(zv.data_ptr(), stride, npix, C, s.data_ptr(), q.data_ptr(), scr.data_ptr(), scr.numel(), st) == 0
    out = dict(scale=f32(C), shift=f32(C), mean=f32(C), invstd=f32(C), rm=bn["rm"].clone(), rv=bn["rv"].clone())
    scr.fill_(float("nan"))
    assert L.y5obb_bn_batch_stats(zv.data_ptr(), stride, npix, C, bn["gamma"].data_ptr(), bn["beta"].data_ptr(), EPS, MOM,
                                  out["rm"].data_ptr(), out["rv"].data_ptr(), out["scale"].data_ptr(),
                                  out["shift"].data_ptr(), out["mean"].data_ptr(), out["invstd"].data_ptr(),
                                  scr.data_ptr(), scr.numel(), st) == 0
    torch.cuda.synchronize()
    return s, q, out


STAT_CASES = [(C, w, r) for C in STAT_C for w, r in (("2", 10), ("lanes-1", 10), ("full-1", 0), ("full+1", 100))
              if not (w == "lanes-1" and bnref.stat_layout(C)[2] < 2)]


@pytest.mark.parametrize("C,which,ratio", STAT_CASES)
def test_bn_stats(C, which, ratio):
    """Sums within the summation bound, finalised statistics from the kernel's own sums, quality against fp64."""
    npix = stat_npix(C, which)
    g = torch.Generator(device=DEV).manual_seed(C * 7 + npix)
    zbuf, zv = slab((npix,), C, extra=16, c_off=8, fill=IN_SENT)
    zv.copy_(gen_z((npix,), C, ratio, g))
    bn = rand_bn(C, g)
    s, q, out = run_stats(zv, zbuf.shape[-1], npix, C, bn)
    check_sums(zv, npix, C, s, q, "bn_stats sums")
    check_batch_stats(zv, npix, C, s, q, bn, out, ratio, "bn_batch_stats")


@pytest.mark.parametrize("ratio", [0, 10, 100, 300])
def test_bn_stats_full_layer(ratio):
    """The stem's BatchNorm of the benchmarked plan: 8 x 512 x 512 pixels, 48 channels, in a wider buffer."""
    npix, C = 8 * 512 * 512, 48
    g = torch.Generator(device=DEV).manual_seed(ratio)
    zbuf, zv = slab((npix,), C, extra=16, c_off=8, fill=IN_SENT)
    zv.copy_(gen_z((npix,), C, ratio, g))
    bn = rand_bn(C, g)
    s, q, out = run_stats(zv, zbuf.shape[-1], npix, C, bn)
    check_sums(zv, npix, C, s, q, "bn_stats sums")
    check_batch_stats(zv, npix, C, s, q, bn, out, ratio, "bn_batch_stats")


APPLY_SHAPES = [(2, 5, 7, 48), (1, 3, 3, 2056), (2, 16, 24, 384), (1, 1, 1, 8), (3, 9, 11, 96)]


APPLY_FLAGS = [(a, r, u) for a in (0, 1) for r in (0, 1) for u in (0, 1)]


@pytest.mark.parametrize("shape", APPLY_SHAPES)
@pytest.mark.parametrize("act,res,up", APPLY_FLAGS)
def test_bn_silu_apply(shape, act, res, up):
    B, H, W, C = shape
    g = torch.Generator(device=DEV).manual_seed(B * H * W + C)
    npix = B * H * W
    zbuf, zv = slab((B, H, W), C, extra=16, c_off=8, fill=IN_SENT)
    zv.copy_(gen_z((B, H, W), C, 2.0, g))
    bn = rand_bn(C, g)
    _, _, st = run_stats(zv, zbuf.shape[-1], npix, C, bn)
    rbuf = rv = None
    if res:
        rbuf, rv = slab((B, H, W), C, extra=24, c_off=16, fill=IN_SENT)
        rv.copy_(torch.randn(B, H, W, C, device=DEV, generator=g).bfloat16())
    ybuf, yv = slab((B, H, W), C, extra=32, c_off=24)
    y_before = ybuf.clone()
    ubuf = u_before = None
    if up:
        ubuf, _ = slab((B, 2 * H, 2 * W), C, extra=8, c_off=8)
        u_before = ubuf.clone()
    rc = lib().y5obb_bn_silu_apply(zv.data_ptr(), zbuf.shape[-1], npix, C, W, st["scale"].data_ptr(), st["shift"].data_ptr(),
                                   act, rv.data_ptr() if res else None, rbuf.shape[-1] if res else 0, yv.data_ptr(),
                                   ybuf.shape[-1], ubuf[..., 8:].data_ptr() if up else None, ubuf.shape[-1] if up else 0,
                                   stream())
    assert rc == 0
    torch.cuda.synchronize()
    check_apply(zv, st["scale"], st["shift"], act, rv, yv, ybuf, y_before, 24, (ubuf, u_before, 8) if up else None,
                "bn_silu_apply")


BWD_CASES = [
    # C, npix kind, |mean|/sigma, act, gres (None / 0 overwrite / 1 accumulate), param_accumulate
    (8, "2", 10, 1, 1, 1), (16, "lanes-1", 0, 1, 0, 0), (48, "full+1", 100, 1, 1, 0), (96, "full-1", 10, 0, None, 1),
    (384, "full+1", 0, 1, 1, 1), (768, "lanes-1", 100, 1, 0, 0), (1280, "full-1", 10, 1, None, 0),
    (2056, "full+1", 10, 1, 1, 1), (2056, "2", 100, 0, 0, 0), (48, "8x512x512", 0, 1, 1, 0),
    (48, "8x512x512", 10, 1, 0, 1), (48, "8x512x512", 100, 1, None, 0),
]


@pytest.mark.parametrize("C,which,ratio,act,gmode,pacc", BWD_CASES)
def test_bn_silu_bwd(C, which, ratio, act, gmode, pacc):
    npix = 8 * 512 * 512 if which == "8x512x512" else stat_npix(C, which)
    g = torch.Generator(device=DEV).manual_seed(C + npix + ratio)
    zbuf, zv = slab((npix,), C, extra=16, c_off=8, fill=IN_SENT)
    zv.copy_(gen_z((npix,), C, ratio, g))
    bn = rand_bn(C, g)
    _, _, st = run_stats(zv, zbuf.shape[-1], npix, C, bn)
    dbuf, dyv = slab((npix,), C, extra=8, c_off=0, fill=IN_SENT)
    dyv.copy_(torch.randn(npix, C, device=DEV, generator=g).bfloat16())
    dzbuf, dzv = slab((npix,), C, extra=24, c_off=16)
    dz_before = dzbuf.clone()
    gbuf = gv = None
    if gmode is not None:
        gbuf, gv = slab((npix,), C, extra=16, c_off=8)
        if gmode:
            gv.copy_(torch.randn(npix, C, device=DEV, generator=g).bfloat16())
    g_before = gbuf.clone() if gbuf is not None else None
    s1, s2 = f32(C), f32(C)
    dg, db = torch.randn(C, device=DEV, generator=g), torch.randn(C, device=DEV, generator=g)
    odg, odb = dg.clone(), db.clone()
    scr = scratch(C)
    rc = lib().y5obb_bn_silu_bwd(zv.data_ptr(), zbuf.shape[-1], dyv.data_ptr(), dbuf.shape[-1], npix, C,
                                 st["scale"].data_ptr(), st["shift"].data_ptr(), st["mean"].data_ptr(), st["invstd"].data_ptr(),
                                 act, s1.data_ptr(), s2.data_ptr(), dzv.data_ptr(), dzbuf.shape[-1],
                                 gv.data_ptr() if gv is not None else None, gbuf.shape[-1] if gbuf is not None else 0,
                                 int(gmode or 0), dg.data_ptr(), db.data_ptr(), pacc, scr.data_ptr(), scr.numel(), stream())
    assert rc == 0
    torch.cuda.synchronize()
    unchanged(dzbuf, dz_before, chan_mask(dzbuf, 16, C), "bn_silu_bwd dz")
    if gbuf is not None:
        unchanged(gbuf, g_before, chan_mask(gbuf, 8, C), "bn_silu_bwd gres")
    check_bwd(zv, dyv, st, act, s1, s2, dzv, (gv, g_before[..., 8:8 + C], bool(gmode)) if gbuf is not None else None,
              (dg, db, odg, odb, pacc), "bn_silu_bwd")


UPSAMPLE_SHAPES = [(2, 5, 7, 16), (1, 1, 1, 8), (2, 8, 12, 2056), (3, 4, 3, 96)]


@pytest.mark.parametrize("B,H,W,C", UPSAMPLE_SHAPES)
@pytest.mark.parametrize("acc", [0, 1])
def test_upsample2x_bwd(B, H, W, C, acc):
    g = torch.Generator(device=DEV).manual_seed(B + H + W + C)
    sbuf, sv = slab((B, 2 * H, 2 * W), C, extra=16, c_off=8, fill=IN_SENT)
    sv.copy_(torch.randn(B, 2 * H, 2 * W, C, device=DEV, generator=g).bfloat16())
    dbuf, dv = slab((B, H, W), C, extra=24, c_off=16)
    if acc:
        dv.copy_(torch.randn(B, H, W, C, device=DEV, generator=g).bfloat16())
    want = bnref.upsample2x_bwd_ref(sv, dv.clone() if acc else None)
    s_before, d_before = sbuf.clone(), dbuf.clone()
    assert lib().y5obb_upsample2x_bwd(sv.data_ptr(), sbuf.shape[-1], dv.data_ptr(), dbuf.shape[-1], B * H * W, C, W, acc,
                                      stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(bits(dv), bits(want)), "upsample2x_bwd"
    unchanged(dbuf, d_before, chan_mask(dbuf, 16, C), "upsample2x_bwd")
    assert torch.equal(sbuf, s_before)
    note("upsample2x_bwd (bitwise)", 0.0)


ADD_CASES = [(37, 24, 40, 8), (5, 13, 16, 3), (4096, 96, 128, 16), (1, 8, 8, 0)]


@pytest.mark.parametrize("npix,C,stride,c_off", ADD_CASES)
@pytest.mark.parametrize("acc", [0, 1])
def test_add_f32_to_bf16(npix, C, stride, c_off, acc):
    g = torch.Generator(device=DEV).manual_seed(npix + C)
    src = torch.randn(npix, C, device=DEV, generator=g) * 3
    dbuf = torch.full((npix, stride), OUT_SENT, dtype=torch.bfloat16, device=DEV)
    dv = dbuf[:, c_off:c_off + C]
    if acc:
        dv.copy_(torch.randn(npix, C, device=DEV, generator=g).bfloat16())
    want = (src + dv.float()).bfloat16() if acc else src.bfloat16()
    before = dbuf.clone()
    assert lib().y5obb_add_f32_to_bf16(src.data_ptr(), dv.data_ptr(), stride, npix, C, acc, stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(bits(dv), bits(want)), "add_f32_to_bf16"
    unchanged(dbuf, before, chan_mask(dbuf, c_off, C), "add_f32_to_bf16")
    note("add_f32_to_bf16 (bitwise)", 0.0)


PACK_SHAPES = [(2, 3, 5, 7, 200, 208), (1, 3, 4, 4, 21, 24), (2, 2, 3, 5, 20, 24), (1, 3, 1, 1, 7, 7)]


@pytest.mark.parametrize("B,na,H,W,no,bn", PACK_SHAPES)
def test_detect_grad_pack(B, na, H, W, no, bn):
    """The vec4 path (no, bn multiples of 4) and the one-channel path (odd no); padding channels written as 0."""
    gsrc = torch.Generator(device=DEV).manual_seed(no)
    g = torch.randn(B, na, H, W, no, device=DEV, generator=gsrc)
    n = B * H * W * na * bn
    flat = torch.full((n + 64,), OUT_SENT, dtype=torch.bfloat16, device=DEV)
    assert lib().y5obb_detect_grad_pack(g.data_ptr(), flat.data_ptr(), B, na, H, W, no, bn, stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(bits(flat[:n].view(B, H, W, na * bn)), bits(bnref.detect_grad_pack_ref(g, bn))), "detect_grad_pack"
    assert (flat[n:] == OUT_SENT).all(), "detect_grad_pack wrote past its output"
    note("detect_grad_pack (bitwise)", 0.0)


POOL_SHAPES = [(2, 7, 9, 24), (1, 3, 4, 16), (1, 1, 1, 8), (2, 5, 5, 40), (1, 2, 11, 8), (2, 13, 6, 136)]


POOL_FORMS = ["f32", "bf16", "f32+bf16"]


@pytest.mark.parametrize("B,H,W,C", POOL_SHAPES)
@pytest.mark.parametrize("form", POOL_FORMS)
def test_maxpool5_bwd(B, H, W, C, form):
    """Small-integer activations (ties everywhere), dyadic gradients (fp32 atomics exact in any order): bit for bit against
    ATen's first-maximum routing, added onto what the fp32 buffer held."""
    g = torch.Generator(device=DEV).manual_seed(B * H * W * C)
    xbuf, xv = slab((B, H, W), C, extra=16, c_off=8, fill=IN_SENT)
    xv.copy_(torch.randint(-3, 4, (B, H, W, C), device=DEV, generator=g).bfloat16())
    g32 = (torch.randint(-8, 9, (B, H, W, C), device=DEV, generator=g) / 8.0) if "f32" in form else None
    gbuf, g16 = slab((B, H, W), C, extra=8, c_off=8, fill=IN_SENT)
    g16.copy_((torch.randint(-8, 9, (B, H, W, C), device=DEV, generator=g) / 4.0).bfloat16())
    use16 = "bf16" in form
    gin = torch.randint(-4, 5, (B, H, W, C), device=DEV, generator=g) / 4.0
    gsum = (g32 if g32 is not None else 0) + (g16.float() if use16 else 0)
    want = gin.double() + bnref.maxpool5_route(xv, gsum)
    assert lib().y5obb_maxpool5_bwd(xv.data_ptr(), xbuf.shape[-1], g32.data_ptr() if g32 is not None else None,
                                    g16.data_ptr() if use16 else None, gbuf.shape[-1], gin.data_ptr(), B, H, W, C,
                                    stream()) == 0
    torch.cuda.synchronize()
    bad = bits(gin) != bits(want.float())
    assert not bad.any(), f"maxpool5_bwd: {int(bad.sum())} of {gin.numel()} differ, first at {bad.nonzero()[:4].tolist()}"
    note("maxpool5_bwd (bitwise)", 0.0)


# =========================================================================================================== 2. the plans
PLANS = [pytest.param("m", 8, 1024, 1024, id="yolov5m-b8-1024"),
         pytest.param("s", 2, 256, 320, id="yolov5s-b2-256x320")]


class _Recorder:
    """Stands in for the library during one _forward_eager: records (name, args) and launches nothing."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def rec(*args):
            self.calls.append((name, args))
            return 0
        return rec


def _plan(size, B, H, W, freeze=None, arena_hw=None):
    """The yolov5{size} train plan at B x H x W.  freeze: train.py --freeze (freeze_layers; the backward plan is then built
    for the requires_grad flags it leaves); arena_hw: carve the plan from an arena reserved for B x arena_hw, as train.py
    --multi-scale does."""
    m = build_mirror(size, nc=15, seed=0).train().to(DEV)
    if freeze is not None:
        freeze_layers(m, [freeze] if isinstance(freeze, int) else list(freeze))
    arena = m.reserve_train_arena(B, *arena_hw, DEV) if arena_hw is not None else None
    return m, TrainEngine(m, B, H, W, DEV, arena=arena)


def _trainable(m):
    return tuple(p.requires_grad for p in m.parameters())


def _randomise_bn(m, g):
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                C = mod.num_features
                mod.weight.copy_(0.5 + torch.rand(C, device=DEV, generator=g))
                mod.bias.copy_(0.3 * torch.randn(C, device=DEV, generator=g))
                mod.running_mean.copy_(torch.randn(C, device=DEV, generator=g))
                mod.running_var.copy_(0.5 + torch.rand(C, device=DEV, generator=g))


@pytest.mark.parametrize("size,B,H,W", PLANS)
def test_plan_forward_bn_launches(size, B, H, W, freeze=None, arena_hw=None):
    plan_forward_bn_launches(size, B, H, W, freeze, arena_hw)


def plan_forward_bn_launches(size, B, H, W, freeze=None, arena_hw=None):
    """Every bn_batch_stats / bn_silu_apply pair of the train plan, issued with the arguments _forward_eager passes, on
    controlled z (|mean| / sigma cycling through 0, 3, 10) with every other element of the destination buffers a sentinel.
    -> the number of BatchNorm layers."""
    m, eng = _plan(size, B, H, W, freeze, arena_hw)
    g = torch.Generator(device=DEV).manual_seed(5)
    _randomise_bn(m, g)
    real = eng._L
    rec = _Recorder()
    eng._L = rec
    try:
        eng._forward_eager(torch.zeros(B, 3, H, W, device=DEV))
    finally:
        eng._L = real
    stats = [a for n, a in rec.calls if n == "y5obb_bn_batch_stats"]
    apply = [a for n, a in rec.calls if n == "y5obb_bn_silu_apply"]
    lays = eng.conv_layers
    assert len(stats) == len(apply) == len(lays)
    L, st = lib(), stream()
    n_y2x = n_res = 0
    for i, (lay, sa, aa) in enumerate(zip(lays, stats, apply)):
        kind = f"plan {size} bn"
        z, y = lay.z, lay.y
        npix, C = z.B * z.H * z.W, z.C
        ratio = (0, 3, 10)[i % 3]
        z.buf.fill_(IN_SENT)
        z.view().copy_(gen_z((z.B, z.H, z.W), C, ratio, g))
        bnm = lay.mod.bn
        bn = dict(gamma=bnm.weight.detach().clone(), beta=bnm.bias.detach().clone(), rm=bnm.running_mean.clone(),
                  rv=bnm.running_var.clone())
        s, q = f32(C), f32(C)
        eng.scratch.fill_(float("nan"))
        assert L.y5obb_bn_stats(sa[0], sa[1], sa[2], sa[3], s.data_ptr(), q.data_ptr(), eng.scratch.data_ptr(),
                                eng.scratch.numel(), st) == 0
        eng.scratch.fill_(float("nan"))
        assert L.y5obb_bn_batch_stats(*sa) == 0
        torch.cuda.synchronize()
        out = dict(scale=lay.scale, shift=lay.shift, mean=lay.mean, invstd=lay.invstd, rm=bnm.running_mean,
                   rv=bnm.running_var)
        check_sums(z.view(), npix, C, s, q, f"{kind} sums")
        check_batch_stats(z.view(), npix, C, s, q, bn, out, ratio, f"{kind} stats")
        bufs = {y.buf.data_ptr()} | ({lay.res.buf.data_ptr()} if lay.res else set()) | \
            ({lay.y2x.buf.data_ptr()} if lay.y2x else set())
        assert len(bufs) == 1 + bool(lay.res) + bool(lay.y2x) and z.buf.data_ptr() not in bufs
        y.buf.fill_(OUT_SENT)
        if lay.res is not None:
            n_res += 1
            lay.res.buf.fill_(IN_SENT)
            lay.res.view().copy_(torch.randn(lay.res.view().shape, device=DEV, generator=g).bfloat16())
        y2x = None
        if lay.y2x is not None:
            n_y2x += 1
            lay.y2x.buf.fill_(OUT_SENT)
            y2x = (lay.y2x.buf, lay.y2x.buf.clone(), lay.y2x.c_off)
        y_before = y.buf.clone()
        assert L.y5obb_bn_silu_apply(*aa) == 0
        torch.cuda.synchronize()
        check_apply(z.view(), lay.scale, lay.shift, lay.act, lay.res.view() if lay.res else None, y.view(), y.buf, y_before,
                    y.c_off, y2x, f"{kind}_silu_apply")
    print(f"\n{size} b{B} {H}x{W}: {len(lays)} BatchNorm layers' forward launches checked ({n_res} with a residual, "
          f"{n_y2x} with a 2x copy)")
    assert n_y2x > 0 and n_res > 0
    return len(lays)


def _defaults(fn):
    return {k: p.default for k, p in inspect.signature(fn).parameters.items() if p.default is not inspect.Parameter.empty}


def _consumers(m, H, W):
    """id(Conv module) -> how many gradient contributions its output receives, from the model graph: a top-level output
    gets one per consuming Conv / SPPF / Upsample / Detect, two per C3 (cv1 and cv2 both read it), and what its Concat gets;
    inside a C3 / SPPF the counts follow the block's structure.  A consumer counts only where the plan produces its data
    gradient: into the output of a layer whose gradient is needed (layout.grad_liveness under the model's requires_grad
    flags; a frozen module's parameters all freeze together, so its inner convs share its liveness).  Every other output
    gets none."""
    mods = list(m.model)
    ch, _ = shapes(mods, H, W)
    live, _ = grad_liveness(mods, ch, lambda mm: any(p.requires_grad for p in mm.parameters()))
    users = {}
    for mm in mods:
        for s in sources(mm):
            users.setdefault(s, []).append(mm)

    def E(i):
        if i not in live:
            return 0
        n = 0
        for mm in users.get(i, []):
            n += E(mm.i) if _is(mm, "Concat") else (2 if _is(mm, "C3") else 1)
        return n

    cnt = {}
    for mm in mods:
        on = int(mm.i in live)
        if _is(mm, "Conv"):
            cnt[id(mm)] = E(mm.i)
        elif _is(mm, "C3"):
            cnt[id(mm.cv3)] = E(mm.i)
            cnt[id(mm.cv1)] = on * (1 + int(mm.m[0].add))
            cnt[id(mm.cv2)] = on
            for j, bt in enumerate(mm.m):
                cnt[id(bt.cv1)] = on
                cnt[id(bt.cv2)] = on * (1 + int(mm.m[j + 1].add) if j + 1 < len(mm.m) else on)
        elif _is(mm, "SPPF"):
            cnt[id(mm.cv2)] = E(mm.i)
            cnt[id(mm.cv1)] = 2 * on   # cv2's data gradient of the whole concat, then the pool chain's add
    return cnt


@pytest.mark.parametrize("size,B,H,W", PLANS)
def test_plan_backward_steps(size, B, H, W, freeze=None, arena_hw=None):
    plan_backward_steps(size, B, H, W, freeze, arena_hw)


def plan_backward_steps(size, B, H, W, freeze=None, arena_hw=None):
    """Every non-conv step of BackwardPlan.steps alone through its own closure on sentinel-filled buffers, against section
    1's references; then the accumulate flags of every gradient range in step order.  -> (step kinds, the number of
    gradient ranges whose flags were checked)."""
    m, eng = _plan(size, B, H, W, freeze, arena_hw)
    plan = BackwardPlan(eng, _trainable(m))
    g = torch.Generator(device=DEV).manual_seed(9)
    _randomise_bn(m, g)
    L, st = lib(), stream()
    det = m.model[-1]
    kinds = {}
    pools = {p.cat4.data_ptr(): p for p in eng.layers if isinstance(p, _PoolLayer)}
    for tag, fn in plan.steps:
        if tag in ("dgrad", "wgrad", "zero"):
            continue
        a = _defaults(fn)
        kinds[tag] = kinds.get(tag, 0) + 1
        kind = f"plan {size} {tag}"
        if tag == "detect_pack":
            gin = plan.det_grads_in[a["l"]]
            gin.copy_(torch.randn(gin.shape, device=DEV, generator=g))
            a["dzd"].fill_(OUT_SENT)
            fn(st)
            torch.cuda.synchronize()
            assert torch.equal(bits(a["dzd"]), bits(bnref.detect_grad_pack_ref(gin, a["bn"]))), kind
        elif tag == "detect_bias":
            dzd, n, C = a["dzd"], a["n"], a["C"]
            dzd.copy_(torch.randn(dzd.shape, device=DEV, generator=g).bfloat16())
            a["s1"].fill_(float("nan"))
            a["s2"].fill_(float("nan"))
            eng.scratch.fill_(float("nan"))
            fn(st)
            torch.cuda.synchronize()
            check_sums(dzd, n, C, a["s1"], a["s2"], kind)
        elif tag == "upsample_bwd":
            g2, gy, acc = a["g2"], a["gy"], a["acc"]
            g2.buf.fill_(IN_SENT)
            g2.view().copy_(torch.randn(g2.view().shape, device=DEV, generator=g).bfloat16())
            gy.buf.fill_(OUT_SENT)
            if acc:
                gy.view().copy_(torch.randn(gy.view().shape, device=DEV, generator=g).bfloat16())
            want = bnref.upsample2x_bwd_ref(g2.view(), gy.view().clone() if acc else None)
            before, g2_before = gy.buf.clone(), g2.buf.clone()
            fn(st)
            torch.cuda.synchronize()
            assert torch.equal(bits(gy.view()), bits(want)), kind
            unchanged(gy.buf, before, chan_mask(gy.buf, gy.c_off, gy.C), kind)
            assert torch.equal(bits(g2.buf), bits(g2_before)), kind
        elif tag == "pool_bwd":
            cat4, c_ = pools[a["base"]].cat4, pools[a["base"]].c
            gc = plan.gbuf[cat4.data_ptr()]
            assert gc.data_ptr() == a["gbase"]
            cat4.copy_(torch.randint(-3, 4, cat4.shape, device=DEV, generator=g).bfloat16())
            gc.copy_((torch.randint(-8, 9, gc.shape, device=DEV, generator=g) / 8.0).bfloat16())
            for t in (a["t0"], a["t1"], a["t2"]):
                t.fill_(float("nan"))     # the step zeroes them itself
            before = gc.clone()
            sl = [slice(k * c_, (k + 1) * c_) for k in range(4)]
            t2 = bnref.maxpool5_route(cat4[..., sl[2]], gc[..., sl[3]].float())
            t1 = bnref.maxpool5_route(cat4[..., sl[1]], t2 + gc[..., sl[2]].double())
            t0 = bnref.maxpool5_route(cat4[..., sl[0]], t1 + gc[..., sl[1]].double())
            want0 = (t0.float() + before[..., sl[0]].float()).bfloat16()
            fn(st)
            torch.cuda.synchronize()
            for t, w in ((a["t2"], t2), (a["t1"], t1), (a["t0"], t0)):
                assert torch.equal(bits(t), bits(w.float().reshape(-1))), f"{kind}: pool chain stage"
            assert torch.equal(bits(gc[..., sl[0]]), bits(want0)), f"{kind}: pool gradient add"
            unchanged(gc, before, chan_mask(gc, 0, c_), kind)
        elif tag == "bn_bwd":
            lay, z, gy, dz, gres, gacc = a["lay"], a["z"], a["gy"], a["dz"], a["gres"], a["gacc"]
            npix, C = a["npix"], a["C"]
            z.buf.fill_(IN_SENT)
            z.view().copy_(gen_z((z.B, z.H, z.W), C, (0, 3, 10)[kinds[tag] % 3], g))
            bnm = lay.mod.bn
            eng.scratch.fill_(float("nan"))
            assert L.y5obb_bn_batch_stats(z.ptr, z.pix_stride, npix, C, bnm.weight.data_ptr(), bnm.bias.data_ptr(), EPS, MOM,
                                          bnm.running_mean.data_ptr(), bnm.running_var.data_ptr(), lay.scale.data_ptr(),
                                          lay.shift.data_ptr(), lay.mean.data_ptr(), lay.invstd.data_ptr(),
                                          eng.scratch.data_ptr(), eng.scratch.numel(), st) == 0
            gy.buf.fill_(IN_SENT)
            gy.view().copy_((0.5 * torch.randn(gy.view().shape, device=DEV, generator=g)).bfloat16())
            dz.fill_(OUT_SENT)
            if gres is not None:
                gres.buf.fill_(OUT_SENT)
                if gacc:
                    gres.view().copy_(torch.randn(gres.view().shape, device=DEV, generator=g).bfloat16())
                g_before = gres.buf.clone()
            plan.flat.fill_(OUT_SENT)
            flat_before = plan.flat.clone()
            eng.scratch.fill_(float("nan"))
            stt = dict(scale=lay.scale.clone(), shift=lay.shift.clone(), mean=lay.mean.clone(), invstd=lay.invstd.clone())
            fn(st)
            torch.cuda.synchronize()
            dg, db = a["dg"], a["db"]
            fm = torch.zeros(plan.flat.shape, dtype=torch.bool, device=DEV)
            for v in (dg, db):
                o = (v.data_ptr() - plan.flat.data_ptr()) // 4
                fm[o:o + v.numel()] = True
            unchanged(plan.flat, flat_before, fm, f"{kind} flat gradient")
            gr = None
            if gres is not None:
                unchanged(gres.buf, g_before, chan_mask(gres.buf, gres.c_off, gres.C), f"{kind} gres")
                gr = (gres.view(), g_before[..., gres.c_off:gres.c_off + gres.C], bool(gacc))
            check_bwd(z.view(), gy.view(), stt, lay.act, a["s1"], a["s2"], dz, gr,
                      (dg, db, torch.zeros_like(dg), torch.zeros_like(db), 0), kind)   # the plan overwrites dgamma / dbeta
        else:
            raise AssertionError(f"unexpected backward step {tag}")
    need = {"detect_pack", "detect_bias", "upsample_bwd", "bn_bwd"}
    if any(isinstance(lay, _PoolLayer) and i in plan._live_out for i, lay in enumerate(eng.layers)):
        need.add("pool_bwd")      # (a frozen backbone takes SPPF's backward with it)
    assert need <= set(kinds), kinds
    print(f"\n{size} b{B} {H}x{W}: backward steps checked {kinds}")

    # ---- accumulate flags: every contribution to a gradient range, in step order
    ops = {}
    for part in plan.det_parts + plan.conv_parts:
        for op in part.get("dgrad_ops", []):
            ops[op._h.value] = (id(part), op)
    contrib, seen = [], set()
    for tag, fn in plan.steps:
        a = _defaults(fn)
        if tag == "dgrad":
            pid, op = ops[a["h"].value]
            gx, acc = op._keep[3], int(bool(op.desc.res))
            if pid in seen:   # the other phases of a stride-2 data gradient: the same range and flag
                assert contrib[-1][:3] == (gx.buf.data_ptr(), gx.c_off, gx.C) and contrib[-1][3] == acc
                continue
            seen.add(pid)
            contrib.append((gx.buf.data_ptr(), gx.c_off, gx.C, acc, "dgrad"))
        elif tag == "upsample_bwd":
            contrib.append((a["gy"].buf.data_ptr(), a["gy"].c_off, a["gy"].C, int(a["acc"]), tag))
        elif tag == "bn_bwd" and a["gres"] is not None:
            r = a["gres"]
            contrib.append((r.buf.data_ptr(), r.c_off, r.C, int(a["gacc"]), "bn_bwd residual"))
        elif tag == "pool_bwd":
            contrib.append((a["gbase"], 0, a["c_"], 1, "pool add"))
    cnt = _consumers(m, H, W)
    n_checked = 0
    for lay in eng.conv_layers:
        if cnt[id(lay.mod)] == 0:   # pruned: nothing may write its gradient range (if its buffer has a gradient at all)
            gb = plan.gbuf.get(lay.y.buf.data_ptr())
            if gb is not None:
                lo, hi = lay.y.c_off, lay.y.c_off + lay.y.C
                hit = [c for c in contrib if c[0] == gb.data_ptr() and c[1] < hi and lo < c[1] + c[2]]
                assert not hit, f"a pruned {type(lay.mod).__name__} output [{lo}, {hi}) receives gradient: {hit}"
            continue
        gy = plan.gbuf[lay.y.buf.data_ptr()].data_ptr(), lay.y.c_off, lay.y.C
        seq = [(c[3], c[4]) for c in contrib if c[0] == gy[0] and c[1] <= gy[1] and gy[1] + gy[2] <= c[1] + c[2]]
        part = [c for c in contrib if c[0] == gy[0] and c[1] < gy[1] + gy[2] and gy[1] < c[1] + c[2]
                and not (c[1] <= gy[1] and gy[1] + gy[2] <= c[1] + c[2])]
        assert not part, f"partial overlap of a gradient range: {part}"
        want = [0] + [1] * (cnt[id(lay.mod)] - 1)
        assert [f for f, _ in seq] == want, f"gradient of a {type(lay.mod).__name__} output [{gy[1]}, {gy[1] + gy[2]}): " \
                                            f"flags {seq}, want {want}"
        n_checked += 1
    print(f"accumulate flags of {n_checked} gradient ranges match the model graph's consumer counts")
    return kinds, n_checked
