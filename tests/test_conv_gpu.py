"""GPU parity tests for the wgmma implicit-GEMM convolution, through the C ABI.

Floating-point kernel: the reference is plain PyTorch fp32 (F.conv2d on the same bf16-rounded inputs
and weights, then bias / SiLU / residual as models/common.py:37-49,94-104 and the Detect decode of
models/yolo.py:63-81).  Tolerance: the kernel accumulates in fp32 and rounds the result once to bf16,
so |err| <= 2^-8 * |ref| + 2e-2 (the absolute term covers bf16 rounding of the residual sum and the
fast-math SiLU); the Detect head writes fp32 and is held to 2e-3 relative / 2e-3 absolute.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _mk(B, H, W, Ctot, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(B, H, W, Ctot, generator=g) * 1.0).to(torch.bfloat16).to(DEV)


def _ref_conv(x_nhwc, w, b, stride, pad, act, res=None):
    x = x_nhwc.float().permute(0, 3, 1, 2)
    y = F.conv2d(x, w.to(torch.bfloat16).float(), b, stride=stride, padding=pad)
    if act:
        y = y * torch.sigmoid(y)
    y = y.permute(0, 2, 3, 1)
    if res is not None:
        y = y + res.float()
    return y


def _check(got, ref, what):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    tol = ref.abs() * 2 ** -8 + 2e-2
    bad = err > tol
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.numel()} out of tolerance, max err {err.max().item():.4g}"


CASES = [
    # B, H, W, Cin, Cout, k, s, act
    (2, 32, 32, 64, 64, 1, 1, True),      # BK=64, single N tile
    (1, 64, 64, 48, 96, 1, 1, True),      # ragged K chunk (48 of 64 via TMA zero fill)
    (2, 32, 32, 32, 32, 3, 1, True),      # BK=32 (64-byte swizzle), 3x3 halo via OOB
    (2, 64, 64, 64, 128, 3, 2, True),     # stride 2 through tensor-map element strides
    (1, 128, 128, 16, 32, 3, 1, True),    # BK=16 (32-byte swizzle): the stem's space-to-depth form
    (2, 16, 16, 256, 512, 1, 1, True),    # two N tiles, 4 K chunks
    (1, 32, 32, 128, 256, 3, 1, False),   # no activation, BN=256
    (3, 20, 20, 80, 80, 3, 1, True),      # ragged spatial tiles (20 not a tile multiple), 2 K chunks of 64 for 80
    (1, 40, 24, 96, 48, 3, 2, True),      # stride 2, non-square, ragged
    (2, 8, 8, 768, 768, 1, 1, True),      # 3 N tiles x 12 K chunks
]


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,s,act", CASES)
def test_conv_matches_torch_fp32(B, H, W, Cin, Cout, k, s, act):
    from yolov5_obb_b200.conv import Conv, Slice, pack_weights
    pad = k // 2
    g = torch.Generator(device="cpu").manual_seed(Cin * 131 + Cout)
    x = _mk(B, H, W, Cin, 1)
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).to(DEV)
    b = (torch.randn(Cout, generator=g) * 0.1).to(DEV)
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    out = torch.full((B, Ho, Wo, Cout), float("nan"), dtype=torch.bfloat16, device=DEV)
    wp, bp = pack_weights(w, b)
    conv = Conv(Slice.full(x), wp, bp, Cout, k, s, pad, act, out=Slice.full(out))
    conv.run()
    torch.cuda.synchronize()
    _check(out, _ref_conv(x, w, b, s, pad, act), f"conv {Cin}->{Cout} k{k} s{s}")
    info = conv.info()
    assert info["flops"] == 2.0 * B * Ho * Wo * Cout * Cin * k * k


@pytest.mark.parametrize("flags", [1, 2, 3])  # NO_ROWSHIFT, NO_RESIDENT, both: the classic one-load-per-tap path
@pytest.mark.parametrize("Cin,Cout", [(32, 32), (128, 128), (80, 320)])
def test_conv_3x3_streamed_and_classic_paths(flags, Cin, Cout):
    from yolov5_obb_b200.conv import Conv, Slice, pack_weights
    B, H, W = 2, 24, 40
    g = torch.Generator(device="cpu").manual_seed(Cin + flags)
    x = _mk(B, H, W, Cin, 4)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (Cin * 9) ** 0.5).to(DEV)
    b = (torch.randn(Cout, generator=g) * 0.1).to(DEV)
    out = torch.full((B, H, W, Cout), float("nan"), dtype=torch.bfloat16, device=DEV)
    wp, bp = pack_weights(w, b)
    Conv(Slice.full(x), wp, bp, Cout, 3, 1, 1, True, out=Slice.full(out), flags=flags).run()
    torch.cuda.synchronize()
    _check(out, _ref_conv(x, w, b, 1, 1, True), f"3x3 {Cin}->{Cout} flags={flags}")


@pytest.mark.parametrize("flags", [0, 4])  # pixel-pair view vs TMA element strides along W
def test_conv_stride2_slice_paths(flags):
    from yolov5_obb_b200.conv import Conv, Slice, pack_weights
    B, H, W = 2, 32, 48
    buf = _mk(B, H, W, 160, 8)            # input = channels [32, 112): ragged against BK = 64
    g = torch.Generator(device="cpu").manual_seed(21)
    w = (torch.randn(96, 80, 3, 3, generator=g) / (80 * 9) ** 0.5).to(DEV)
    b = (torch.randn(96, generator=g) * 0.1).to(DEV)
    out = torch.full((B, H // 2, W // 2, 96), float("nan"), dtype=torch.bfloat16, device=DEV)
    wp, bp = pack_weights(w, b)
    Conv(Slice(buf, 32, 80), wp, bp, 96, 3, 2, 1, True, out=Slice.full(out), flags=flags).run()
    torch.cuda.synchronize()
    _check(out, _ref_conv(buf[..., 32:112], w, b, 2, 1, True), f"3x3 s2 slice flags={flags}")


def test_conv_slices_residual_and_upsample():
    """Concat-offset store, strided input slice, Bottleneck residual (in place) and the 2x up-sampled copy."""
    from yolov5_obb_b200.conv import Conv, Slice, pack_weights
    B, H, W = 2, 16, 16
    big_in = _mk(B, H, W, 192, 3)          # input = channels [64,128)
    big_out = torch.zeros((B, H, W, 160), dtype=torch.bfloat16, device=DEV)  # output -> channels [32,96)
    up = torch.zeros((B, 2 * H, 2 * W, 128), dtype=torch.bfloat16, device=DEV)  # up-sampled copy -> [64,128)
    g = torch.Generator(device="cpu").manual_seed(7)
    w = (torch.randn(64, 64, 3, 3, generator=g) / 24).to(DEV)
    b = (torch.randn(64, generator=g) * 0.1).to(DEV)
    wp, bp = pack_weights(w, b)
    xin = Slice(big_in, 64, 64)
    res = Slice(big_out, 32, 64)
    big_out[..., 32:96] = _mk(B, H, W, 64, 5)  # residual lives where the result goes (in-place chain)
    res_copy = big_out[..., 32:96].clone()
    conv = Conv(xin, wp, bp, 64, 3, 1, 1, True, out=Slice(big_out, 32, 64), res=res, out2x=Slice(up, 64, 64))
    conv.run()
    torch.cuda.synchronize()
    ref = _ref_conv(big_in[..., 64:128], w, b, 1, 1, True, res=res_copy)
    _check(big_out[..., 32:96], ref, "residual slice")
    assert (big_out[..., :32] == 0).all() and (big_out[..., 96:] == 0).all(), "neighbouring channels untouched"
    up_ref = big_out[..., 32:96].repeat_interleave(2, 1).repeat_interleave(2, 2)
    assert torch.equal(up[..., 64:128], up_ref)
    assert (up[..., :64] == 0).all()


@pytest.mark.parametrize("cout,hw", [(32, 40), (64, 24), (256, 16)])
def test_inplace_residual_add(cout, hw):
    """The Bottleneck chain adds in place (out = res): the epilogue loads the residual from the output slice, adds it in fp32
    and stores over it.  The result must match the fp32 reference within the kernel's tolerance, and the channels of the
    wider buffer outside the slice must stay untouched."""
    from yolov5_obb_b200.conv import Conv, Slice, pack_weights
    B, H, W = 2, hw, hw + 8
    g = torch.Generator(device="cpu").manual_seed(11)
    w = (torch.randn(cout, cout, 3, 3, generator=g) / (3 * cout ** 0.5)).to(DEV)
    b = (torch.randn(cout, generator=g) * 0.1).to(DEV)
    wp, bp = pack_weights(w, b)
    x = _mk(B, H, W, cout, 21)
    res0 = _mk(B, H, W, 2 * cout, 22)
    buf = res0.clone()                      # the chain lives in channels [0, cout) of a wider (concat) buffer
    Conv(Slice.full(x), wp, bp, cout, 3, 1, 1, True, out=Slice(buf, 0, cout), res=Slice(buf, 0, cout)).run()
    torch.cuda.synchronize()
    _check(buf[..., :cout], _ref_conv(x, w, b, 1, 1, True, res=res0[..., :cout]), "in-place residual")
    assert torch.equal(buf[..., cout:], res0[..., cout:]), "neighbouring channels untouched"


@pytest.mark.parametrize("decode", [True, False])
def test_detect_head(decode):
    """models/yolo.py:63-81: 1x1 conv -> [B,3,H,W,no] (train) or sigmoid+decode rows of [B, A, no] (eval)."""
    from yolov5_obb_b200.conv import Conv, Slice, pack_weights, MODE_DETECT
    B, H, W, Cin, na, no = 2, 16, 16, 128, 3, 200
    stride = 16.0
    anchors_px = [30., 61., 62., 45., 59., 119.]
    g = torch.Generator(device="cpu").manual_seed(11)
    x = _mk(B, H, W, Cin, 2)
    w = (torch.randn(na * no, Cin, 1, 1, generator=g) / Cin ** 0.5).to(DEV)
    b = (torch.randn(na * no, generator=g)).to(DEV)
    rows_total = na * H * W + 50  # this level sits at row offset 50 of a taller output
    out = torch.full((B, rows_total, no), float("nan"), dtype=torch.float32, device=DEV)
    wp, bp = pack_weights(w, b, MODE_DETECT, no)
    conv = Conv(Slice.full(x), wp, bp, na * no, 1, 1, 0, False,
                det=dict(out=out, rows_per_image=rows_total, row_off=50, no=no, decode=decode, stride=stride,
                         anchors_px=anchors_px))
    conv.run()
    torch.cuda.synchronize()
    y = F.conv2d(x.float().permute(0, 3, 1, 2), w.to(torch.bfloat16).float(), b)           # [B, 600, H, W]
    y = y.view(B, na, no, H, W).permute(0, 1, 3, 4, 2).contiguous()                         # yolo.py:65
    if decode:
        y = y.sigmoid()
        yv, xv = torch.meshgrid(torch.arange(H, device=DEV), torch.arange(W, device=DEV), indexing="ij")
        grid = torch.stack((xv, yv), 2).view(1, 1, H, W, 2).float()
        ag = torch.tensor(anchors_px, device=DEV).view(1, na, 1, 1, 2)
        y[..., 0:2] = (y[..., 0:2] * 2 - 0.5 + grid) * stride
        y[..., 2:4] = (y[..., 2:4] * 2) ** 2 * ag
    ref = y.view(B, -1, no)
    got = out[:, 50:]
    err = (got - ref).abs()
    tol = ref.abs() * 2e-3 + 2e-3
    assert not (err > tol).any(), f"max err {err.max().item()}"
    assert torch.isnan(out[:, :50]).all(), "rows of other levels untouched"


def test_conv_rejects_bad_arguments():
    from yolov5_obb_b200.conv import Conv, Slice, pack_weights
    x = _mk(1, 8, 8, 64, 0)
    wp, bp = pack_weights(torch.zeros(64, 64, 1, 1, device=DEV), None)
    with pytest.raises(RuntimeError):
        Conv(Slice.full(x), wp, bp, 64, 1, 3, 0, True, out=Slice.full(torch.zeros_like(x)))  # stride 3
    with pytest.raises(RuntimeError):
        Conv(Slice.full(x), wp, bp, 64, 1, 1, 0, True, out=None)  # no destination


@pytest.mark.parametrize("H,W,C", [(5, 7, 8), (32, 32, 32), (40, 70, 16)])
def test_sppf_pool_matches_chained_maxpool(H, W, C):
    """models/common.py:190-196: y1 = m(x), y2 = m(y1), y3 = m(y2) with m = MaxPool2d(5, 1, 2), written at channel
    offsets C, 2C, 3C of the same buffer (bit-exact: max is exact in bf16)."""
    from yolov5_obb_b200 import _lib
    B = 2
    buf = torch.zeros((B, H, W, 4 * C + 8), dtype=torch.bfloat16, device=DEV)  # wider than 4C: a slice of a bigger buffer
    x = _mk(B, H, W, C, 12)
    buf[..., :C] = x
    rc = _lib.lib().y5obb_sppf_pool(buf.data_ptr(), buf.shape[3], B, H, W, C, _lib.stream_ptr(torch.device(DEV)))
    assert rc == 0
    torch.cuda.synchronize()
    xn = x.float().permute(0, 3, 1, 2)
    y1 = F.max_pool2d(xn, 5, 1, 2)
    y2 = F.max_pool2d(y1, 5, 1, 2)
    y3 = F.max_pool2d(y2, 5, 1, 2)
    for k, y in enumerate((y1, y2, y3), 1):
        assert torch.equal(buf[..., k * C:(k + 1) * C].float(), y.permute(0, 2, 3, 1)), k
    assert torch.equal(buf[..., :C], x) and (buf[..., 4 * C:] == 0).all()
