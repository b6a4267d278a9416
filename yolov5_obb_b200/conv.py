"""Host-side handle for the wgmma implicit-GEMM convolution (csrc/conv_sm90.cu) behind the C ABI.

A `Slice` names a channel range of an NHWC bf16 (or, in fp16 plans, fp16) buffer; convs read and write slices, which is how
Concat (models/common.py:267-274) disappears: producers store at a channel offset.
"""
import ctypes
from ctypes import c_void_p, c_int, c_int64, c_float, POINTER
from dataclasses import dataclass
from typing import Optional

import torch

from . import _lib

MODE_CONV, MODE_DETECT = 0, 1


class ConvDesc(ctypes.Structure):
    """Mirror of y5obb_conv_desc in include/y5obb.h."""
    _fields_ = [
        ("in_", c_void_p), ("in_pix_stride", c_int64), ("in_row_stride", c_int64), ("in_img_stride", c_int64),
        ("B", c_int), ("Hin", c_int), ("Win", c_int), ("Cin", c_int), ("hbm_cin", c_int),
        ("w", c_void_p), ("bias", c_void_p),
        ("Cout", c_int), ("KH", c_int), ("KW", c_int), ("stride", c_int), ("pad_h", c_int), ("pad_w", c_int),
        ("mode", c_int), ("act", c_int), ("flags", c_int),
        ("out", c_void_p), ("out_pix_stride", c_int64),
        ("res", c_void_p), ("res_pix_stride", c_int64),
        ("out2x", c_void_p), ("out2x_pix_stride", c_int64),
        ("det_out", c_void_p), ("det_rows_per_image", c_int64), ("det_row_off", c_int64),
        ("det_no", c_int), ("det_decode", c_int), ("det_stride", c_float), ("det_anchor", c_float * 6),
        ("out_h", c_int), ("out_w", c_int), ("out_row_stride", c_int64), ("out_img_stride", c_int64),
        ("res_row_stride", c_int64), ("res_img_stride", c_int64),
        ("det_descale", c_int), ("det_inv_scale", c_float), ("det_flip_w", c_float),
    ]


@dataclass
class Slice:
    """Channels [c_off, c_off + C) of an NHWC bf16 or fp16 buffer [B, H, W, Ctot]."""
    buf: torch.Tensor
    c_off: int
    C: int

    def __post_init__(self):
        assert self.buf.dtype in (torch.bfloat16, torch.float16) and self.buf.dim() == 4 and self.buf.is_contiguous()
        assert 0 <= self.c_off and self.c_off + self.C <= self.buf.shape[3]
        assert self.c_off % 8 == 0 and self.buf.shape[3] % 8 == 0, "slices must start on 16-byte boundaries"

    @property
    def ptr(self) -> int:
        return self.buf.data_ptr() + 2 * self.c_off

    @property
    def pix_stride(self) -> int:
        return self.buf.shape[3]

    @property
    def B(self):
        return self.buf.shape[0]

    @property
    def H(self):
        return self.buf.shape[1]

    @property
    def W(self):
        return self.buf.shape[2]

    def view(self) -> torch.Tensor:
        return self.buf[..., self.c_off:self.c_off + self.C]

    @staticmethod
    def full(buf: torch.Tensor) -> "Slice":
        return Slice(buf, 0, buf.shape[3])


def tiling(cin: int, cout: int, mode: int = MODE_CONV, det_no: int = 0):
    """(block_k, block_n, cin_pad, cout_pad, n_tiles_n) — the kernel's own choice (y5obb_conv_tiling)."""
    v = [c_int() for _ in range(5)]
    rc = _lib.lib().y5obb_conv_tiling(cin, cout, mode, det_no, *[ctypes.byref(x) for x in v])
    _lib.check(rc, "y5obb_conv_tiling")
    return tuple(x.value for x in v)


def pack_weights(w: torch.Tensor, bias: Optional[torch.Tensor], mode: int = MODE_CONV, det_no: int = 0,
                 dtype: torch.dtype = torch.bfloat16):
    """[Cout, Cin, KH, KW] fp32 (+ bias [Cout]) -> `dtype` (bf16, or fp16 for the fp16 plans) [KH*KW, cout_pad, cin_pad]
    K-major, fp32 bias [cout_pad + 32].

    Detect mode places anchor a's det_no rows at [a*block_n, a*block_n + det_no) so one N tile == one anchor.
    """
    cout, cin, kh, kw = w.shape
    bk, bn, cin_pad, cout_pad, nt = tiling(cin, cout, mode, det_no)
    wp = torch.zeros((kh * kw, cout_pad, cin_pad), dtype=torch.float32, device=w.device)
    bp = torch.zeros((cout_pad + 32,), dtype=torch.float32, device=w.device)  # epilogue reads bias in 32-wide chunks
    wt = w.detach().float().permute(2, 3, 0, 1).reshape(kh * kw, cout, cin)
    if mode == MODE_DETECT:
        for a in range(nt):
            wp[:, a * bn:a * bn + det_no, :cin] = wt[:, a * det_no:(a + 1) * det_no]
            if bias is not None:
                bp[a * bn:a * bn + det_no] = bias.detach().float()[a * det_no:(a + 1) * det_no]
    else:
        wp[:, :cout, :cin] = wt
        if bias is not None:
            bp[:cout] = bias.detach().float()
    return wp.to(dtype).contiguous(), bp.contiguous()


@dataclass
class WindowView:
    """An input described by explicit strides: `C` channels per position may exceed `pix_stride` (overlapping
    horizontal windows — how the stem's three kw taps become one contiguous K range)."""
    buf: torch.Tensor
    ptr: int
    pix_stride: int
    row_stride: int
    img_stride: int
    B: int
    H: int
    W: int
    C: int
    hbm_c: int = 0


NO_ROWSHIFT, NO_RESIDENT, NO_PAIRW, BIAS_HALVED = 1, 2, 4, 8
ONE_CTA = 64   # one CTA per SM for every instantiation (A/B comparison of the two-CTA plans)
DETECT_GENERIC = 128   # compact Detect records through the shared epilogue (A/B comparison of the records epilogue)
F16 = 256              # fp16 operands and outputs (Y5OBB_CONV_F16): the fp16 inference plans


class Conv:
    """One convolution bound to fixed buffers (TMA descriptors are baked at creation)."""

    def __init__(self, x, w_packed: torch.Tensor, bias_pad: torch.Tensor, cout: int, k, stride: int,
                 pad, act: bool, out: Optional[Slice] = None, res: Optional[Slice] = None,
                 out2x: Optional[Slice] = None, det: Optional[dict] = None, flags: int = 0,
                 out_geom: Optional[dict] = None, bias_prehalved: bool = False):
        """out_geom (optional): dict(h, w, off, pix, row, img) - the output (and the residual, which must then be the same
        slice) has h x w pixels at element offset `off` of the slice with pixel / row / image strides in elements."""
        _lib.require_cuda(x.buf, "conv input")
        kh, kw = (k, k) if isinstance(k, int) else k
        ph, pw = (pad, pad) if isinstance(pad, int) else pad
        d = ConvDesc()
        d.in_, d.in_pix_stride = x.ptr, x.pix_stride
        if isinstance(x, WindowView):
            d.in_row_stride, d.in_img_stride, d.hbm_cin = x.row_stride, x.img_stride, x.hbm_c
        d.B, d.Hin, d.Win, d.Cin = x.B, x.H, x.W, x.C
        if act and not det:
            # the SiLU epilogue evaluates h + h*tanh(h) with h = 0.5*acc + 0.5*bias: hand it 0.5*bias
            if not bias_prehalved:
                bias_pad = (bias_pad * 0.5).contiguous()
            flags |= BIAS_HALVED
        d.w, d.bias = w_packed.data_ptr(), bias_pad.data_ptr()
        d.Cout, d.KH, d.KW, d.stride, d.pad_h, d.pad_w = cout, kh, kw, stride, ph, pw
        d.mode, d.act, d.flags = (MODE_DETECT if det else MODE_CONV), int(bool(act)), flags
        if out is not None:
            d.out, d.out_pix_stride = out.ptr, out.pix_stride
        if res is not None:
            d.res, d.res_pix_stride = res.ptr, res.pix_stride
        if out_geom is not None:
            g = out_geom
            d.out, d.out_pix_stride = out.ptr + 2 * g["off"], g["pix"]
            d.out_h, d.out_w, d.out_row_stride, d.out_img_stride = g["h"], g["w"], g["row"], g["img"]
            if res is not None:
                assert res.ptr == out.ptr, "a strided residual must be the output slice itself (in-place accumulation)"
                d.res, d.res_pix_stride = res.ptr + 2 * g["off"], g["pix"]
                d.res_row_stride, d.res_img_stride = g["row"], g["img"]
        if out2x is not None:
            d.out2x, d.out2x_pix_stride = out2x.ptr, out2x.pix_stride
        if det:
            d.det_out = det["out"].data_ptr()
            d.det_rows_per_image, d.det_row_off = det["rows_per_image"], det["row_off"]
            d.det_no, d.det_decode, d.det_stride = det["no"], int(det["decode"]), float(det["stride"])  # decode 2 = compact records
            d.det_anchor = (c_float * 6)(*[float(v) for v in det["anchors_px"]])
            if det.get("descale") is not None:   # (inv_scale, flip_w): a test-time-augmentation branch (engine.TTAPlan)
                d.det_descale = 1
                d.det_inv_scale, d.det_flip_w = (float(v) for v in det["descale"])
        self._keep = (x, w_packed, bias_pad, out, res, out2x, det)  # buffers must outlive the descriptors
        self.desc = d  # what the kernel was told (tests/convref.py evaluates it)
        self._h = c_void_p()
        with torch.cuda.device(x.buf.device):
            rc = _lib.lib().y5obb_conv_create(ctypes.byref(d), ctypes.byref(self._h))
        _lib.check(rc, "y5obb_conv_create")
        self.device = x.buf.device

    def run(self, stream: Optional[int] = None) -> None:
        rc = _lib.lib().y5obb_conv_run(self._h, stream if stream is not None else _lib.stream_ptr(self.device))
        _lib.check(rc, "y5obb_conv_run")

    def info(self) -> dict:
        fl, by = ctypes.c_double(), ctypes.c_double()
        g, bn, bk, st = c_int(), c_int(), c_int(), c_int()
        _lib.lib().y5obb_conv_info(self._h, ctypes.byref(fl), ctypes.byref(by), ctypes.byref(g), ctypes.byref(bn),
                                   ctypes.byref(bk), ctypes.byref(st))
        cta, res, rs, grp = c_int(), c_int(), c_int(), c_int()
        _lib.lib().y5obb_conv_schedule(self._h, ctypes.byref(cta), ctypes.byref(res), ctypes.byref(rs), ctypes.byref(grp))
        return dict(flops=fl.value, hbm_bytes=by.value, grid=g.value, block_n=bn.value, block_k=bk.value,
                    stages=st.value, ctas_per_sm=cta.value, resident=res.value, rowshift=rs.value, group=grp.value)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                _lib.lib().y5obb_conv_destroy(h)
            except Exception:
                pass
            self._h = None
