"""tests/convref.py against torch's own convolution and its gradients, on descriptor-shaped CPU inputs built the way
conv.Conv / train_ops.Wgrad and the plans fill them: a wrong reference would hide a wrong kernel in
test_conv_plans_exact_gpu.py."""
import ctypes
from types import SimpleNamespace

import torch
import torch.nn.functional as F

from tests.convref import conv_reference, expected, wgrad_reference
from yolov5_obb_b200.conv import BIAS_HALVED, MODE_DETECT, ConvDesc, Slice, WindowView
from yolov5_obb_b200.train_ops import WgradDesc

G = torch.Generator().manual_seed(7)


def ints(*shape, lo=-4, hi=4):
    return torch.randint(lo, hi + 1, shape, generator=G).double()


def nhwc_bf(t):
    return t.permute(0, 2, 3, 1).contiguous().bfloat16()


def fake_conv(x, wp, bp, cout, k, stride, pad, out=None, res=None, out2x=None, det=None, act=False, flags=0, geom=None):
    """The descriptor conv.Conv.__init__ fills, on CPU tensors."""
    d = ConvDesc()
    d.in_, d.in_pix_stride = x.ptr, x.pix_stride
    if isinstance(x, WindowView):
        d.in_row_stride, d.in_img_stride, d.hbm_cin = x.row_stride, x.img_stride, x.hbm_c
    d.B, d.Hin, d.Win, d.Cin = x.B, x.H, x.W, x.C
    d.w, d.bias = wp.data_ptr(), bp.data_ptr()
    (d.KH, d.KW), d.stride, (d.pad_h, d.pad_w) = k, stride, pad
    d.Cout, d.mode, d.act, d.flags = cout, MODE_DETECT if det else 0, int(act), flags
    if out is not None:
        d.out, d.out_pix_stride = out.ptr, out.pix_stride
    if res is not None:
        d.res, d.res_pix_stride = res.ptr, res.pix_stride
    if geom is not None:
        d.out, d.out_pix_stride = out.ptr + 2 * geom["off"], geom["pix"]
        d.out_h, d.out_w, d.out_row_stride, d.out_img_stride = geom["h"], geom["w"], geom["row"], geom["img"]
        if res is not None:
            d.res, d.res_pix_stride = d.out, geom["pix"]
            d.res_row_stride, d.res_img_stride = geom["row"], geom["img"]
    if out2x is not None:
        d.out2x, d.out2x_pix_stride = out2x.ptr, out2x.pix_stride
    if det:
        d.det_out, d.det_rows_per_image, d.det_row_off = det["out"].data_ptr(), det["rows_per_image"], det["row_off"]
        d.det_no, d.det_decode, d.det_stride = det["no"], det["decode"], det["stride"]
        d.det_anchor = (ctypes.c_float * 6)(*det["anchors_px"])
    return SimpleNamespace(desc=d, _keep=(x, wp, bp, out, res, out2x, det))


def pack(w, cin_pad, cout_pad):
    """[Cout, Cin, KH, KW] -> bf16 [KH*KW, cout_pad, cin_pad] (the conv layout)."""
    co, ci, kh, kw = w.shape
    wp = torch.zeros(kh * kw, cout_pad, cin_pad)
    wp[:, :co, :ci] = w.permute(2, 3, 0, 1).reshape(kh * kw, co, ci).float()
    return wp.bfloat16()


def merged(recs):
    assert len(recs) == 1
    return recs[0]


def test_plain_conv_slices_residual_out2x_and_halved_bias():
    B, H, W, Cin, Cout = 2, 6, 10, 24, 16
    xb = torch.full((B, H, W, 40), 4096.0).bfloat16()
    x = ints(B, Cin, H, W)
    xb[..., 8:8 + Cin] = nhwc_bf(x)
    w = ints(Cout, Cin, 3, 3)
    b = ints(Cout)
    bp = torch.zeros(Cout + 32)
    bp[:Cout] = b.float() * 0.5
    ob = torch.full((B, H // 2, W // 2, 32), -3.0).bfloat16()
    r = ints(B, Cout, H // 2, W // 2)
    ob[..., 16:] = nhwc_bf(r)
    up = torch.zeros(B, H, W, 24).bfloat16()
    out = Slice(ob, 16, Cout)
    op = fake_conv(Slice(xb, 8, Cin), pack(w, 24, 16), bp, Cout, (3, 3), 2, (1, 1), out=out, res=out,
                   out2x=Slice(up, 8, Cout), act=True, flags=BIAS_HALVED)
    recs = {rec.buf.data_ptr(): rec for rec in conv_reference(op)}
    pre = F.conv2d(x, w, b, stride=2, padding=1)
    want = (F.silu(pre) + r).permute(0, 2, 3, 1)
    rec = recs[ob.data_ptr()]
    assert rec.mask[..., 16:].all() and not rec.mask[..., :16].any()
    assert torch.allclose(rec.value[..., 16:], want, rtol=1e-12, atol=1e-9)
    assert (rec.tol[..., 16:] >= 2.0 ** -8 * want.abs()).all()
    rec2 = recs[up.data_ptr()]
    assert rec2.mask[..., 8:].all() and not rec2.mask[..., :8].any()
    assert torch.allclose(rec2.value[..., 8:], want.repeat_interleave(2, 1).repeat_interleave(2, 2), rtol=1e-12)


def s2d(img):
    """The stem input layout: x_s2d[b, i, 1 + j, (dy*2+dx)*3 + c] = img[b, c, 2i+dy, 2j+dx], zero pad pixels / channels."""
    B, _, H, W = img.shape
    t = torch.zeros(B, H // 2, W // 2 + 2, 16)
    for dy in range(2):
        for dx in range(2):
            t[:, :, 1:-1, (dy * 2 + dx) * 3:(dy * 2 + dx) * 3 + 3] = img[:, :, dy::2, dx::2].permute(0, 2, 3, 1).float()
    return t.bfloat16()


def stem_weight(w):
    """[Cout, 3, 6, 6] -> [Cout, 48, 3, 1]: tap ty, column tx * 16 + (dy*2+dx)*3 + c."""
    w2 = torch.zeros(w.shape[0], 16, 3, 3, dtype=w.dtype)
    for dy in range(2):
        for dx in range(2):
            w2[:, (dy * 2 + dx) * 3:(dy * 2 + dx) * 3 + 3] = w[:, :, dy::2, dx::2]
    return w2.permute(0, 3, 1, 2).reshape(w.shape[0], 48, 3, 1)


def test_stem_window_view_conv_and_wgrad():
    """The overlapping 48-channel window (pixel stride 16) equals the 6x6 / stride 2 / pad 2 convolution of the image, and
    its weight gradient that of the image conv, re-mapped."""
    B, H, W, Cout = 2, 12, 16, 16
    img = ints(B, 3, H, W)
    xs = s2d(img)
    Wp = W // 2 + 2
    win = WindowView(buf=xs, ptr=xs.data_ptr(), pix_stride=16, row_stride=Wp * 16, img_stride=(H // 2) * Wp * 16,
                     B=B, H=H // 2, W=W // 2, C=48, hbm_c=16)
    w = ints(Cout, 3, 6, 6)
    ob = torch.zeros(B, H // 2, W // 2, Cout).bfloat16()
    op = fake_conv(win, pack(stem_weight(w), 48, Cout), torch.zeros(Cout + 32), Cout, (3, 1), 1, (1, 0), out=Slice.full(ob))
    rec = merged(conv_reference(op))
    want = F.conv2d(img, w, stride=2, padding=2).permute(0, 2, 3, 1)
    assert rec.mask.all() and torch.equal(rec.value, want)

    dz = ints(B, Cout, H // 2, W // 2)
    dzb = nhwc_bf(dz)
    dw = ints(3 * Cout * 48).float()
    before = dw.clone()
    d = WgradDesc(dzb.data_ptr(), Cout, xs.data_ptr(), 16, Wp * 16, (H // 2) * Wp * 16, dw.data_ptr(), 0, 0, 0,
                  B, Cout, H // 2, W // 2, 48, H // 2, W // 2, 3, 1, 1, 1, 0, 0, 0)
    rec = merged(wgrad_reference(SimpleNamespace(desc=d, _keep=(dw, dzb, xs))))
    g = torch.nn.grad.conv2d_weight(img, (Cout, 3, 6, 6), dz, stride=2, padding=2)
    want = before.double().view(3, Cout, 48) + stem_weight(g)[..., 0].permute(2, 0, 1)  # [ty][co][tx*16 + ch]
    assert rec.mask.all() and torch.equal(rec.value.view(3, Cout, 48), want)


def test_out_geom_parity_writes_compose_the_stride2_dgrad():
    """Four 1- / 2-tap convolutions of dz, each written to one pixel parity of gx through out_geom (the phase form of the
    stride-2 data gradient), accumulated onto gx: together conv2d_input of the 3x3 / stride 2 / pad 1 forward weight."""
    B, Ho, Wo, Cout, C = 2, 3, 5, 16, 24
    Hi, Wi = 2 * Ho, 2 * Wo
    w = ints(Cout, C, 3, 3)
    dz = ints(B, Cout, Ho, Wo)
    dzb = nhwc_bf(dz)
    g0 = ints(B, C, Hi, Wi)
    gb = torch.full((B, Hi, Wi, 40), 7.0).bfloat16()
    gb[..., 8:8 + C] = nhwc_bf(g0)
    gx = Slice(gb, 8, C)
    ps = gx.pix_stride
    value, mask = torch.zeros(gb.shape, dtype=torch.float64), torch.zeros(gb.shape, dtype=torch.bool)
    for ph in range(2):
        for pw in range(2):
            kh2, kw2 = (2 if ph else 1), (2 if pw else 1)
            wd = torch.zeros(C, Cout, kh2, kw2, dtype=torch.float64)
            for th in range(kh2):
                for tw in range(kw2):
                    skh = (2 if th == 0 else 0) if ph else 1
                    skw = (2 if tw == 0 else 0) if pw else 1
                    wd[:, :, th, tw] = w[:, :, skh, skw].t()
            geom = dict(h=Ho, w=Wo, off=(ph * Wi + pw) * ps, pix=2 * ps, row=2 * Wi * ps, img=Hi * Wi * ps)
            op = fake_conv(Slice.full(dzb), pack(wd, Cout, C), torch.zeros(C + 32), C, (kh2, kw2), 1, (0, 0), out=gx,
                           res=gx, geom=geom)
            rec = merged(conv_reference(op))
            par = torch.zeros(Hi, Wi, dtype=torch.bool)
            par[ph::2, pw::2] = True
            assert torch.equal(rec.mask[..., 8:8 + C], par.view(1, Hi, Wi, 1).expand(B, Hi, Wi, C))
            assert not rec.mask[..., :8].any() and not rec.mask[..., 8 + C:].any() and not (mask & rec.mask).any()
            mask |= rec.mask
            value[rec.mask] = rec.value[rec.mask]
    want = g0 + torch.nn.grad.conv2d_input((B, C, Hi, Wi), w, dz, stride=2, padding=1)
    assert mask[..., 8:8 + C].all() and torch.equal(value[..., 8:8 + C], want.permute(0, 2, 3, 1))


def detect_pack(w, b, na, no, bn, cin_pad):
    """Anchor a's `no` rows at [a*bn, a*bn + no) of the packed weights and bias (one N tile per anchor)."""
    wp = torch.zeros(1, na * bn, cin_pad)
    bp = torch.zeros(na * bn + 32)
    for a in range(na):
        wp[0, a * bn:a * bn + no, :w.shape[1]] = w[a * no:(a + 1) * no, :, 0, 0].float()
        bp[a * bn:a * bn + no] = b[a * no:(a + 1) * no].float()
    return wp.bfloat16(), bp


def test_detect_anchor_gaps_raw_decoded_and_records():
    """Detect rows at row_off, one anchor per N tile at a*block_n (gap rows hold weights that must not be read), raw logits,
    the sigmoid / grid / anchor decode, and compact records whose theta index is the FIRST maximum."""
    B, H, W, Cin, na, nc = 2, 3, 5, 32, 3, 3
    no = 5 + nc + 180
    bn = (no + 15) // 16 * 16
    x = ints(B, Cin, H, W, lo=-1, hi=1)
    xb = nhwc_bf(x)
    w = ints(na * no, Cin, 1, 1, lo=-1, hi=1) * (torch.rand(na * no, Cin, 1, 1, generator=G) < 0.1)
    b = ints(na * no, lo=-2, hi=2)
    wp, bp = detect_pack(w, b, na, no, bn, Cin)
    for a in range(na):  # the gap rows: a kernel that read them would differ
        wp[0, a * bn + no:(a + 1) * bn, :] = 3.0
    pre = F.conv2d(x, w, b).view(B, na, no, H, W).permute(0, 1, 3, 4, 2)      # [B, na, H, W, no]
    rows_total, row_off = na * H * W + 8, 8
    stride, anchors = 8.0, [10.0, 13.0, 16.0, 30.0, 33.0, 23.0]
    for decode in (0, 1, 2):
        rw = no if decode < 2 else (nc + 6 + 3) // 4 * 4
        out = torch.full((B, rows_total, rw), -5.0)
        det = dict(out=out, rows_per_image=rows_total, row_off=row_off, no=no, decode=decode, stride=stride,
                   anchors_px=anchors)
        rec = merged(conv_reference(fake_conv(Slice.full(xb), wp, bp, na * no, (1, 1), 1, (0, 0), det=det)))
        m = torch.zeros(B, rows_total, rw, dtype=torch.bool)
        m[:, row_off:] = True
        assert torch.equal(rec.mask, m)
        got = rec.value[:, row_off:].view(B, na, H, W, rw)
        if decode == 0:
            assert rec.tol is None and torch.equal(got, pre)
            continue
        s = torch.sigmoid(pre)
        gx = torch.arange(W).view(1, 1, 1, W)
        gy = torch.arange(H).view(1, 1, H, 1)
        anc = torch.tensor(anchors, dtype=torch.float64).view(1, na, 1, 1, 2)
        dec = torch.cat([(s[..., :1] * 2 - 0.5 + gx.unsqueeze(-1)) * stride, (s[..., 1:2] * 2 - 0.5 + gy.unsqueeze(-1)) * stride,
                         (s[..., 2:4] * 2) ** 2 * anc, s[..., 4:]], -1)
        if decode == 1:
            assert torch.allclose(got, dec, rtol=1e-12, atol=1e-12)
            continue
        nfix = 5 + nc
        assert torch.allclose(got[..., :nfix], dec[..., :nfix], rtol=1e-12, atol=1e-12)
        assert (got[..., nfix + 1:] == 0).all() and (rec.tol.view(B, rows_total, rw)[:, row_off:, nfix:] == 0).all()
        lg = pre[..., nfix:].reshape(-1, 180).tolist()
        first = [row.index(max(row)) for row in lg]
        assert got[..., nfix].flatten().tolist() == first
        assert rec.ties > 0, "small integer logits must tie"


def test_co_group_wgrad_parameter_layout():
    """Detect's weight gradient: dz has na padded groups of bn channels, dW is the [na*no, Cin, 1, 1] parameter layout, the
    gap channels of dz (filled here) are skipped; accumulated onto what dW held."""
    B, H, W, Cin, na, no = 2, 3, 5, 24, 3, 20
    bn = 32
    dz = ints(B, na * bn, H, W)
    x = ints(B, Cin, H, W)
    xb = torch.full((B, H, W, 40), 4096.0).bfloat16()
    xb[..., 16:16 + Cin] = nhwc_bf(x)
    flat = ints(na * no * Cin + 64).float()
    dw = flat[32:32 + na * no * Cin].view(na * no, Cin, 1, 1)
    before = flat.clone()
    dzb = nhwc_bf(dz)
    d = WgradDesc(dzb.data_ptr(), na * bn, xb.data_ptr() + 2 * 16, 40, 0, 0, dw.data_ptr(), 1, Cin, 1,
                  B, na * bn, H, W, Cin, H, W, 1, 1, 1, 0, 0, no, bn)
    rec = merged(wgrad_reference(SimpleNamespace(desc=d, _keep=(dw, dzb, xb, flat))))
    assert rec.buf is flat
    m = torch.zeros(flat.shape, dtype=torch.bool)
    m[32:32 + na * no * Cin] = True
    assert torch.equal(rec.mask, m)
    real = dz.view(B, na, bn, H, W)[:, :, :no].reshape(B, na * no, H, W)
    want = before[32:32 + na * no * Cin].double() + torch.nn.grad.conv2d_weight(x, (na * no, Cin, 1, 1), real).flatten()
    assert torch.equal(rec.value[m], want)
    assert torch.equal(expected(rec)[m], want.float())


def test_strided_wgrad_taps_layout_and_ragged_edge():
    """[taps][Cout][Cin] layout, stride 2 over a channel slice whose output map does not cover the input's last row."""
    B, Hi, Wi, Cin, Cout = 2, 7, 9, 24, 16
    Ho, Wo = (Hi + 2 - 3) // 2 + 1, (Wi + 2 - 3) // 2 + 1
    x = ints(B, Cin, Hi, Wi)
    dz = ints(B, Cout, Ho, Wo)
    xb = torch.full((B, Hi, Wi, 32), 4096.0).bfloat16()
    xb[..., 8:] = nhwc_bf(x)
    dzb = nhwc_bf(dz)
    dw = torch.zeros(9 * Cout * Cin)
    d = WgradDesc(dzb.data_ptr(), Cout, xb.data_ptr() + 16, 32, 0, 0, dw.data_ptr(), 0, 0, 0,
                  B, Cout, Ho, Wo, Cin, Hi, Wi, 3, 3, 2, 1, 1, 0, 0)
    rec = merged(wgrad_reference(SimpleNamespace(desc=d, _keep=(dw, dzb, xb))))
    g = torch.nn.grad.conv2d_weight(x, (Cout, Cin, 3, 3), dz, stride=2, padding=1)
    assert rec.mask.all() and torch.equal(rec.value.view(9, Cout, Cin), g.permute(2, 3, 0, 1).reshape(9, Cout, Cin))
