"""fp64 references of one conv launch (yolov5_obb_b200.conv.Conv) and one weight-gradient launch (train_ops.Wgrad),
evaluated from what the kernel was told: the ctypes descriptor the op keeps as `.desc`, read through its own pointers,
strides and extents on the buffers the op keeps alive.

For integer-valued operands only: every operand must hold integers, and the caller keeps the sum of |a*b| over each
reduction below 2^24 (exact in fp32).  The library's fp64 convolution then differs from the exact integer by far less than
0.5 whatever algorithm it picks, so the reference rounds it to the nearest integer and is exact.

Each reference returns `Written` records, one per destination buffer: the elements the op writes (`mask`), their exact value
before the store's rounding to the buffer's type (`value`), and, where the epilogue approximates (SiLU, Detect sigmoid), a
per-element bound `tol` of that approximation and of the store's rounding (0 where the element must match bit for bit after
the rounding).  Everything outside `mask` must be left unchanged.
"""
from dataclasses import dataclass
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

# tanh.approx.f32: maximum relative error 2^-11 (PTX ISA, "tanh"); the bound uses twice that
TANH_REL = 2.0 ** -10
F32_REL = 2.0 ** -24        # one fp32 rounding, relative
BF16_REL = 2.0 ** -8        # one bf16 rounding to nearest: half an ulp is at most 2^-8 of the value


@dataclass
class Written:
    buf: torch.Tensor                    # a destination tensor the op keeps (contiguous)
    mask: torch.Tensor                   # bool, buf's shape: the elements the op writes
    value: torch.Tensor                  # float64, buf's shape: their exact value (0 outside mask)
    tol: Optional[torch.Tensor] = None   # float64, buf's shape, or None: every written element is bitwise
    ties: int = 0                        # Detect records: rows whose 180 theta logits have a tied maximum


def expected(w: Written) -> torch.Tensor:
    """The exact value stored in the buffer's type: fp64 -> fp32 (exact for integers below 2^24) -> one rounding to
    nearest-even."""
    return w.value.float().to(w.buf.dtype)


def view_at(buf: torch.Tensor, ptr: int, shape, strides) -> torch.Tensor:
    """The strided view a descriptor describes, as a view of `buf` (must lie inside it)."""
    esz = buf.element_size()
    off = ptr - buf.data_ptr()
    assert off >= 0 and off % esz == 0, "descriptor pointer outside its buffer"
    off //= esz
    last = off + sum((n - 1) * s for n, s in zip(shape, strides))
    assert buf.is_contiguous() and last < buf.numel(), "descriptor extent runs past its buffer"
    return torch.as_strided(buf, tuple(shape), tuple(strides), buf.storage_offset() + off)


def _mask_view(mask: torch.Tensor, buf: torch.Tensor, ptr: int, shape, strides) -> torch.Tensor:
    off = (ptr - buf.data_ptr()) // buf.element_size()
    return torch.as_strided(mask, tuple(shape), tuple(strides), off)


class _Dest:
    """Accumulates Written records per destination buffer (an op may write several places of one buffer)."""

    def __init__(self):
        self.w: Dict[int, Written] = {}

    def put(self, buf, ptr, shape, strides, value, tol=None):
        key = buf.data_ptr()
        if key not in self.w:
            self.w[key] = Written(buf, torch.zeros(buf.shape, dtype=torch.bool, device=buf.device),
                                  torch.zeros(buf.shape, dtype=torch.float64, device=buf.device), None)
        rec = self.w[key]
        mv = _mask_view(rec.mask, buf, ptr, shape, strides)
        assert not mv.any(), "the op writes one element twice"
        mv.fill_(True)
        _mask_view(rec.value, buf, ptr, shape, strides).copy_(value)
        if tol is not None:
            if rec.tol is None:
                rec.tol = torch.zeros(buf.shape, dtype=torch.float64, device=buf.device)
            _mask_view(rec.tol, buf, ptr, shape, strides).copy_(tol)

    def out(self) -> List[Written]:
        return list(self.w.values())


def _integer(t: torch.Tensor, what: str) -> torch.Tensor:
    assert torch.isfinite(t).all() and torch.equal(t, t.round()), f"{what} must hold integers"
    return t


def _conv_nchw(x, w, stride, pad, out_hw):
    """x [B, Cin, H, W], w [Cout, Cin, KH, KW] (fp64, integers) -> [B, Cout, Ho, Wo]: zeros outside the input, exactly
    out_hw outputs (the kernel reads past the far edge as zeros when the descriptor asks for more)."""
    (ph, pw), (Ho, Wo) = pad, out_hw
    KH, KW = w.shape[2:]
    H, W = x.shape[2:]
    xp = F.pad(x, (pw, (Wo - 1) * stride + KW - pw - W, ph, (Ho - 1) * stride + KH - ph - H))
    return F.conv2d(xp, w, stride=stride).round()


def conv_reference(op) -> List[Written]:
    """Everything one Conv launch writes, from op.desc and op._keep = (x, w_packed, bias_pad, out, res, out2x, det)."""
    from yolov5_obb_b200.conv import BIAS_HALVED, MODE_DETECT
    d = op.desc
    x, wp, bp, out, res, out2x, det = op._keep
    B, Hin, Win, Cin, Cout, KH, KW, s = d.B, d.Hin, d.Win, d.Cin, d.Cout, d.KH, d.KW, d.stride
    ps = d.in_pix_stride
    rs = d.in_row_stride or ps * Win
    ims = d.in_img_stride or rs * Hin
    xin = _integer(view_at(x.buf, d.in_, (B, Hin, Win, Cin), (ims, rs, ps, 1)).double(), "input")
    geom = d.out_h > 0
    Hout = d.out_h if geom else (Hin + 2 * d.pad_h - KH) // s + 1
    Wout = d.out_w if geom else (Win + 2 * d.pad_w - KW) // s + 1

    # packed weights [KH*KW, cout_pad, cin_pad]: output channel co lives in row rows[co]
    assert d.w == wp.data_ptr() and d.bias == bp.data_ptr() and wp.shape[0] == KH * KW
    detect = d.mode == MODE_DETECT
    if detect:
        na, no = Cout // d.det_no, d.det_no
        bn = wp.shape[1] // na
        rows = torch.tensor([a * bn + j for a in range(na) for j in range(no)], device=wp.device)
    else:
        rows = torch.arange(Cout, device=wp.device)
    w = wp[:, rows, :Cin].double().view(KH, KW, Cout, Cin).permute(2, 3, 0, 1)
    bias = bp[rows].double() * (2.0 if d.flags & BIAS_HALVED else 1.0)
    _integer(w, "weights")
    _integer(bias, "bias")

    acc = _conv_nchw(xin.permute(0, 3, 1, 2), w.contiguous(), s, (d.pad_h, d.pad_w), (Hout, Wout))
    pre = acc.permute(0, 2, 3, 1) + bias        # [B, Hout, Wout, Cout], exact
    dest = _Dest()
    if not detect:
        tol = None
        if d.act:  # y = h + h tanh(h), h = 0.5 pre: tanh.approx's error times |h|, and the fma's rounding
            h = 0.5 * pre
            y = pre * torch.sigmoid(pre)
            tol = h.abs() * torch.tanh(h).abs() * TANH_REL + F32_REL * (y.abs() + h.abs())
        else:
            y = pre
        if d.res:
            rps = d.res_pix_stride
            rrs = d.res_row_stride if geom else rps * Wout
            ris = d.res_img_stride if geom else rps * Wout * Hout
            y = y + _integer(view_at(res.buf, d.res, (B, Hout, Wout, Cout), (ris, rrs, rps, 1)).double(), "residual")
        if tol is not None:  # the fp32 sum with the residual, then one bf16 rounding of the perturbed value
            tol = tol * (1 + BF16_REL) + (2 * F32_REL + BF16_REL) * y.abs()
        ops_ = d.out_pix_stride
        ors = d.out_row_stride if geom else ops_ * Wout
        ois = d.out_img_stride if geom else ops_ * Wout * Hout
        dest.put(out.buf, d.out, (B, Hout, Wout, Cout), (ois, ors, ops_, 1), y, tol)
        if d.out2x:
            px = d.out2x_pix_stride
            y2 = y.repeat_interleave(2, 1).repeat_interleave(2, 2)
            t2 = tol.repeat_interleave(2, 1).repeat_interleave(2, 2) if tol is not None else None
            dest.put(out2x.buf, d.out2x, (B, 2 * Hout, 2 * Wout, Cout), (4 * Hout * Wout * px, 2 * Wout * px, px, 1), y2, t2)
        return dest.out()

    # Detect: row b * rows_per_image + row_off + (a * Hout + h) * Wout + w of the fp32 output
    nfix = no - 180
    rec_w = (nfix + 1 + 3) // 4 * 4
    rw = rec_w if d.det_decode == 2 else no
    p5 = pre.view(B, Hout, Wout, na, no).permute(0, 3, 1, 2, 4)   # [B, na, H, W, no]
    tol, ties = None, 0
    if d.det_decode == 0:
        val = p5
    else:
        sig = torch.sigmoid(p5)
        # sigmoid = fma(0.5, tanh.approx(0.5 x), 0.5): half of tanh's error, one fp32 rounding
        es = 0.5 * TANH_REL * torch.tanh(0.5 * p5).abs() + F32_REL
        gx = torch.arange(Wout, device=pre.device, dtype=torch.float64).view(1, 1, 1, Wout)
        gy = torch.arange(Hout, device=pre.device, dtype=torch.float64).view(1, 1, Hout, 1)
        anc = torch.tensor(list(d.det_anchor), dtype=torch.float64, device=pre.device).view(na, 2)
        st = d.det_stride
        val = sig.clone()
        tol = es.clone()
        val[..., 0] = (sig[..., 0] * 2 - 0.5 + gx) * st
        val[..., 1] = (sig[..., 1] * 2 - 0.5 + gy) * st
        tol[..., 0] = 2 * st * es[..., 0]
        tol[..., 1] = 2 * st * es[..., 1]
        for c in (2, 3):
            a_ = anc[:, c - 2].view(1, na, 1, 1)
            val[..., c] = (sig[..., c] * 2) ** 2 * a_
            tol[..., c] = 8 * a_ * es[..., c] * (1 + es[..., c])
        tol = tol * (1 + 1e-6) + 4 * F32_REL * (val.abs() + st)   # the fp32 roundings of the decode arithmetic
        if d.det_descale:  # test-time augmentation: x y w h times the fp32 1 / s, then x = flip_w - x (two more roundings)
            inv = d.det_inv_scale   # (the descriptor's fp32 value)
            val[..., :4] *= inv
            tol[..., :4] = tol[..., :4] * inv * (1 + F32_REL) + F32_REL * val[..., :4].abs()
            if d.det_flip_w > 0:
                val[..., 0] = d.det_flip_w - val[..., 0]
                tol[..., 0] = tol[..., 0] * (1 + F32_REL) + F32_REL * val[..., 0].abs()
        if d.det_decode == 2:
            theta = p5[..., nfix:].argmax(-1).double()   # the FIRST maximum (torch.argmax's documented rule)
            rec = torch.zeros(val.shape[:-1] + (rec_w,), dtype=torch.float64, device=pre.device)
            rt = torch.zeros_like(rec)
            rec[..., :nfix], rt[..., :nfix] = val[..., :nfix], tol[..., :nfix]
            rec[..., nfix] = theta
            lg = p5[..., nfix:]
            ties = int(((lg == lg.max(-1, keepdim=True).values).sum(-1) > 1).sum())
            val, tol = rec, rt
    R, off = d.det_rows_per_image, d.det_row_off
    buf = det["out"]
    dest.put(buf, d.det_out + 4 * off * rw, (B, na, Hout, Wout, rw),
             (R * rw, Hout * Wout * rw, Wout * rw, rw, 1), val, tol)
    recs = dest.out()
    recs[0].ties = ties
    return recs


def wgrad_reference(wg) -> List[Written]:
    """What one Wgrad launch leaves in its weight-gradient buffer: the values there before the launch plus
    dW[tap][co][ci] = sum over (b, ho, wo) of dz[b, ho, wo, co] * x[b, s*ho + kh - ph, s*wo + kw - pw, ci], at element
    tap * s_tap + row(co) * s_co + ci * s_ci ([taps][Cout][Cin] unless the descriptor gives strides); with co_group =
    (real, padded), channel a * padded + c (c < real) is row a * real + c and the others are not written.
    x may be an overlapping-window view (explicit row / image strides)."""
    d = wg.desc
    tensors = [t for t in wg._keep if isinstance(t, torch.Tensor)]

    def owner(ptr, dtype):  # the largest kept tensor of that type containing ptr
        c = [t for t in tensors if t.dtype == dtype and t.is_contiguous()
             and t.data_ptr() <= ptr < t.data_ptr() + t.numel() * t.element_size()]
        assert c, "descriptor pointer in no kept buffer"
        return max(c, key=lambda t: t.numel())

    B, Cout, Ho, Wo, Cin, Hi, Wi = d.B, d.Cout, d.Ho, d.Wo, d.Cin, d.Hi, d.Wi
    KH, KW, s = d.KH, d.KW, d.stride
    dzp = d.dz_pix_stride
    dz = view_at(owner(d.dz, torch.bfloat16), d.dz, (B, Ho, Wo, Cout), (dzp * Wo * Ho, dzp * Wo, dzp, 1))
    xps = d.x_pix_stride
    xrs = d.x_row_stride or xps * Wi
    xis = d.x_img_stride or xrs * Hi
    x = view_at(owner(d.x, torch.bfloat16), d.x, (B, Hi, Wi, Cin), (xis, xrs, xps, 1))
    g = torch.zeros((Cout, Cin, KH, KW), dtype=torch.float64, device=dz.device)
    for b in range(B):  # per image: fp64 partial sums of integers are exact, so the chunks add exactly
        xb = _integer(x[b:b + 1].double(), "x").permute(0, 3, 1, 2)
        dzb = _integer(dz[b:b + 1].double(), "dz").permute(0, 3, 1, 2).contiguous()
        xb = F.pad(xb, (d.pad_w, (Wo - 1) * s + KW - d.pad_w - Wi, d.pad_h, (Ho - 1) * s + KH - d.pad_h - Hi))
        g += torch.nn.grad.conv2d_weight(xb, g.shape, dzb, stride=s).round()
    if d.co_group_pad:
        na = Cout // d.co_group_pad
        g = g.view(na, d.co_group_pad, Cin, KH, KW)[:, :d.co_group].reshape(na * d.co_group, Cin, KH, KW)
    rows = g.shape[0]
    if d.dw_tap_stride or d.dw_co_stride or d.dw_ci_stride:
        st_tap, st_co, st_ci = d.dw_tap_stride, d.dw_co_stride, d.dw_ci_stride
    else:
        st_tap, st_co, st_ci = Cout * Cin, Cin, 1
    buf = owner(d.dw, torch.float32)
    shape, strides = (rows, Cin, KH * KW), (st_co, st_ci, st_tap)
    before = _integer(view_at(buf, d.dw, shape, strides).double(), "dW before the launch")
    dest = _Dest()
    dest.put(buf, d.dw, shape, strides, before + g.reshape(rows, Cin, KH * KW))
    return dest.out()
