"""GPU parity of the training-only kernels against torch autograd (fp32 on the same bf16-rounded inputs):
BatchNorm(train)+SiLU backward, NHWC->NCHW copies (plain and de-interleaved), tensor-core wgrad."""
import pytest
import torch
import torch.nn.functional as F

from yolov5_obb_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _bf(t):
    return t.to(torch.bfloat16)


@pytest.mark.parametrize("shape", [(2, 12, 16, 48), (3, 67, 50, 16), (2, 40, 64, 320)])
@pytest.mark.parametrize("act,with_res", [(True, False), (True, True), (False, False)])
def test_bn_silu_forward_backward(act, with_res, shape):
    L = _lib.lib()
    st = _lib.stream_ptr(torch.device(DEV))
    B, H, W, C = shape
    g = torch.Generator().manual_seed(3)
    z = _bf(torch.randn(B, H, W, C, generator=g) * 1.5 + 0.3).to(DEV)
    res = _bf(torch.randn(B, H, W, C, generator=g)).to(DEV) if with_res else None
    dy = _bf(torch.randn(B, H, W, C, generator=g)).to(DEV)
    gamma = (torch.rand(C, generator=g) + 0.5).to(DEV)
    beta = (torch.randn(C, generator=g) * 0.2).to(DEV)
    rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    npix = B * H * W
    f32 = lambda: torch.empty(C, dtype=torch.float32, device=DEV)
    s1, s2, scale, shift, mean, invstd = f32(), f32(), f32(), f32(), f32(), f32()
    y = torch.zeros_like(z)
    scr = torch.empty(int(L.y5obb_bn_scratch_floats(C)), dtype=torch.float32, device=DEV)
    assert L.y5obb_bn_stats(z.data_ptr(), C, npix, C, s1.data_ptr(), s2.data_ptr(), scr.data_ptr(), scr.numel(), st) == 0
    s1b, s2b = f32(), f32()   # deterministic: a second pass gives the same bits
    assert L.y5obb_bn_stats(z.data_ptr(), C, npix, C, s1b.data_ptr(), s2b.data_ptr(), scr.data_ptr(), scr.numel(), st) == 0
    torch.cuda.synchronize()
    assert torch.equal(s1, s1b) and torch.equal(s2, s2b)
    assert torch.allclose(s1, z.float().sum((0, 1, 2)), rtol=1e-4, atol=1e-2)
    assert torch.allclose(s2, (z.float() ** 2).sum((0, 1, 2)), rtol=1e-4, atol=1e-2)
    assert L.y5obb_bn_finalize(s1.data_ptr(), s2.data_ptr(), npix, C, gamma.data_ptr(), beta.data_ptr(), 1e-3, 0.03,
                               rm.data_ptr(), rv.data_ptr(), scale.data_ptr(), shift.data_ptr(), mean.data_ptr(),
                               invstd.data_ptr(), st) == 0
    assert L.y5obb_bn_silu_apply(z.data_ptr(), C, npix, C, W, scale.data_ptr(), shift.data_ptr(), int(act),
                                 res.data_ptr() if with_res else None, C, y.data_ptr(), C, None, 0, st) == 0
    # reference (fp32 autograd on the same bf16 values)
    zr = z.float().permute(0, 3, 1, 2).clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    rm_r, rv_r = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    u = F.batch_norm(zr, rm_r, rv_r, gr, br, True, 0.03, 1e-3)
    yr = F.silu(u) if act else u
    if with_res:
        yr = yr + res.float().permute(0, 3, 1, 2)
    torch.cuda.synchronize()
    assert (y.float() - yr.permute(0, 2, 3, 1)).abs().max().item() < 0.03 * yr.abs().max().item() + 0.02
    assert torch.allclose(rm, rm_r, atol=1e-4) and torch.allclose(rv, rv_r, rtol=1e-3, atol=1e-4)
    yr.backward(dy.float().permute(0, 3, 1, 2))
    dz = torch.zeros_like(z)
    gres = torch.zeros_like(z) if with_res else None
    dgam, dbet = f32(), f32()
    rc = L.y5obb_bn_silu_bwd(z.data_ptr(), C, dy.data_ptr(), C, npix, C, scale.data_ptr(), shift.data_ptr(),
                             mean.data_ptr(), invstd.data_ptr(), int(act), s1.data_ptr(), s2.data_ptr(), dz.data_ptr(), C,
                             gres.data_ptr() if with_res else None, C, 0, dgam.data_ptr(), dbet.data_ptr(), 0,
                             scr.data_ptr(), scr.numel(), st)
    assert rc == 0
    torch.cuda.synchronize()
    ref_dz = zr.grad.permute(0, 2, 3, 1)
    assert (dz.float() - ref_dz).abs().max().item() < 0.02 * ref_dz.abs().max().item() + 1e-3
    assert torch.allclose(dgam, gr.grad, rtol=2e-3, atol=2e-2) and torch.allclose(dbet, br.grad, rtol=2e-3, atol=2e-2)
    if with_res:
        assert torch.equal(gres, dy)


WG_CASES = [
    # B, Cin, Cout, H, W, k, s, x_extra, dz_extra (channels of padding around the slices)
    (2, 64, 64, 16, 64, 1, 1, 0, 0),
    (2, 32, 48, 32, 32, 3, 1, 0, 0),
    (1, 128, 256, 16, 16, 3, 1, 64, 0),
    (2, 64, 128, 32, 64, 3, 2, 0, 32),
    (3, 320, 160, 8, 8, 1, 1, 0, 0),
    (2, 48, 96, 24, 40, 3, 2, 16, 16),
    (2, 16, 32, 20, 12, 3, 1, 0, 0),
    (1, 512, 512, 4, 4, 3, 1, 0, 0),
    (2, 80, 40, 10, 6, 1, 1, 8, 8),
]


@pytest.mark.parametrize("B,Cin,Cout,H,W,k,s,xe,ze", WG_CASES)
def test_wgrad_matches_autograd(B, Cin, Cout, H, W, k, s, xe, ze):
    """wgmma wgrad straight from NHWC slices == autograd's conv2d weight gradient on the same bf16-rounded operands."""
    from yolov5_obb_b200.train_ops import Wgrad
    p = k // 2
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    g = torch.Generator().manual_seed(Cin + Cout)
    xbuf = _bf(torch.randn(B, H, W, Cin + 2 * xe, generator=g)).to(DEV)
    zbuf = _bf(torch.randn(B, Ho, Wo, Cout + 2 * ze, generator=g)).to(DEV)
    x, dz = xbuf[..., xe:xe + Cin], zbuf[..., ze:ze + Cout]
    dw = torch.zeros((k * k, Cout, Cin), dtype=torch.float32, device=DEV)
    wg = Wgrad(zbuf.data_ptr() + 2 * ze, zbuf.shape[3], xbuf.data_ptr() + 2 * xe, xbuf.shape[3], dw, B, Cout, Ho, Wo, Cin, H, W,
               k, s, p, keep=(xbuf, zbuf))
    wg.run()
    torch.cuda.synchronize()
    w = torch.zeros((Cout, Cin, k, k), device=DEV, requires_grad=True)
    y = F.conv2d(x.float().permute(0, 3, 1, 2), w, None, s, p)
    y.backward(dz.float().permute(0, 3, 1, 2))
    ref = w.grad.permute(2, 3, 0, 1).reshape(k * k, Cout, Cin)
    err = (dw - ref).abs().max().item()
    assert err < 2e-3 * ref.abs().max().item() + 1e-3, f"max err {err} vs scale {ref.abs().max().item()}"
    wg.run()  # accumulates
    torch.cuda.synchronize()
    assert (dw - 2 * ref).abs().max().item() < 4e-3 * ref.abs().max().item() + 2e-3


def test_wgrad_param_layout_and_padded_groups():
    """dW written straight in the nn.Conv2d layout [Cout][Cin][KH][KW]; Detect's padded per-anchor channel groups."""
    from yolov5_obb_b200.train_ops import Wgrad
    g = torch.Generator().manual_seed(77)
    B, Cin, Cout, H, W, k = 2, 48, 80, 12, 20, 3
    x = _bf(torch.randn(B, H, W, Cin, generator=g)).to(DEV)
    dz = _bf(torch.randn(B, H, W, Cout, generator=g)).to(DEV)
    dw = torch.zeros((Cout, Cin, k, k), dtype=torch.float32, device=DEV)
    Wgrad(dz.data_ptr(), Cout, x.data_ptr(), Cin, dw, B, Cout, H, W, Cin, H, W, k, 1, 1, keep=(x, dz), param_layout=True).run()
    w = torch.zeros((Cout, Cin, k, k), device=DEV, requires_grad=True)
    F.conv2d(x.float().permute(0, 3, 1, 2), w, None, 1, 1).backward(dz.float().permute(0, 3, 1, 2))
    torch.cuda.synchronize()
    assert (dw - w.grad).abs().max().item() < 2e-3 * w.grad.abs().max().item() + 1e-3
    # 3 anchors x 200 real channels padded to 208
    na, no, bn, Cin = 3, 200, 208, 64
    dzp = _bf(torch.randn(B, H, W, na * bn, generator=g)).to(DEV)
    x = _bf(torch.randn(B, H, W, Cin, generator=g)).to(DEV)
    dw = torch.zeros((na * no, Cin, 1, 1), dtype=torch.float32, device=DEV)
    Wgrad(dzp.data_ptr(), na * bn, x.data_ptr(), Cin, dw, B, na * bn, H, W, Cin, H, W, 1, 1, 0, keep=(x, dzp), param_layout=True,
          co_group=(no, bn)).run()
    real = dzp.view(B, H, W, na, bn)[..., :no].reshape(B, H, W, na * no)
    w = torch.zeros((na * no, Cin, 1, 1), device=DEV, requires_grad=True)
    F.conv2d(x.float().permute(0, 3, 1, 2), w).backward(real.float().permute(0, 3, 1, 2))
    torch.cuda.synchronize()
    assert (dw - w.grad).abs().max().item() < 2e-3 * w.grad.abs().max().item() + 1e-3


def test_pack_plan_matches_host_packing():
    """One-launch device packing (csrc/pack_weights.cu) == conv.pack_weights on the host-side formulas, every kind."""
    from yolov5_obb_b200.conv import pack_weights, MODE_DETECT, tiling
    from yolov5_obb_b200.layout import stem_weight
    from yolov5_obb_b200.train_ops import (PackPlan, PACK_FWD, PACK_DGRAD, PACK_STEM, PACK_DETECT, PACK_DETECT_DGRAD,
                                           PACK_DETECT_BIAS)
    g = torch.Generator().manual_seed(3)
    ent, want = [], []

    def add(kind, src, ref, g_real=0, g_pad=0):
        dst = torch.full_like(ref, 7.0)
        ent.append((kind, src, dst, g_real, g_pad))
        want.append(ref)

    for cout, cin, k in [(48, 24, 3), (96, 40, 1), (256, 128, 3), (80, 16, 3)]:
        w = torch.randn(cout, cin, k, k, generator=g).to(DEV)
        add(PACK_FWD, w, pack_weights(w, None)[0])
        add(PACK_DGRAD, w, pack_weights(w.permute(1, 0, 2, 3).flip(2, 3).contiguous(), None)[0])
    w = torch.randn(48, 3, 6, 6, generator=g).to(DEV)
    add(PACK_STEM, w, pack_weights(stem_weight(w), None)[0])
    na, no, cin = 3, 200, 192
    w = torch.randn(na * no, cin, 1, 1, generator=g).to(DEV)
    b = torch.randn(na * no, generator=g).to(DEV)
    wp, bp = pack_weights(w, b, MODE_DETECT, no)
    bn = tiling(cin, na * no, MODE_DETECT, no)[1]
    add(PACK_DETECT, w, wp, no, bn)
    add(PACK_DETECT_BIAS, b, bp, no, bn)
    wT = torch.zeros((cin, na * bn), device=DEV)
    for a in range(na):
        wT[:, a * bn:a * bn + no] = w.view(na, no, cin)[a].t()
    add(PACK_DETECT_DGRAD, w, pack_weights(wT.view(cin, na * bn, 1, 1), None)[0], no, bn)
    from yolov5_obb_b200.train_ops import PACK_DGRAD_S2
    w = torch.randn(96, 48, 3, 3, generator=g).to(DEV)          # stride-2 data gradient, one packing per output parity
    for ph in range(2):
        for pw in range(2):
            kh = [2, 0] if ph else [1]
            kw = [2, 0] if pw else [1]
            sub = w[:, :, kh][:, :, :, kw]                       # [Cout, Cin, KH', KW'] in tap order
            add(PACK_DGRAD_S2, w, pack_weights(sub.permute(1, 0, 2, 3).contiguous(), None)[0], ph * 2 + pw, 0)
    PackPlan(ent, DEV).run()
    torch.cuda.synchronize()
    for (kind, src, dst, _, _), ref in zip(ent, want):
        assert torch.equal(dst, ref), (kind, tuple(src.shape))
