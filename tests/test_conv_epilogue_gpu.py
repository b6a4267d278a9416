"""The conv epilogue at every instruction width N = 16 ... 256, exactly: with and without a residual (added in place, as the
Bottleneck chain does), with and without SiLU, on ragged image edges and ragged output channels, into a channel slice of
a wider buffer, and with the 2x up-sampled copy.  Each launch is checked by test_conv_plans_exact_gpu.check_conv against
tests/convref.py's fp64 reference on integer operands: bit for bit without SiLU, within the SiLU bound with it, and
every element outside the written slice unchanged."""
import pytest
import torch

from tests.test_conv_plans_exact_gpu import DEV, _stats, check_conv
from yolov5_obb_b200.conv import Conv, Slice, pack_weights, tiling

pytestmark = pytest.mark.gpu

# Cout -> the kernel's instruction N: 16, 32, 64 (48: 16 columns never stored), 64, 96 (80), 96, 128, 160 (144), 192,
# 224 (208), 256, and 160 in two N tiles (320)
COUTS = [16, 32, 48, 64, 80, 96, 128, 144, 192, 208, 256, 320]
CIN, B, H, W = 32, 2, 19, 27   # 19 x 27: every tile shape leaves ragged tiles at the bottom and right edges


def instr_n(cout):
    bn = tiling(CIN, cout)[1]
    return 16 if bn <= 16 else (bn + 31) // 32 * 32


def make_conv(cout, k, act, res, up):
    g = torch.Generator(device="cpu").manual_seed(cout)
    w = torch.randn(cout, CIN, k, k, generator=g).to(DEV)   # check_conv replaces weights, bias and activations by integers
    wp, bp = pack_weights(w, torch.randn(cout, generator=g).to(DEV))
    x = torch.zeros(B, H, W, CIN, dtype=torch.bfloat16, device=DEV)
    out = Slice(torch.zeros(B, H, W, cout + 24, dtype=torch.bfloat16, device=DEV), 8, cout)
    up2 = Slice(torch.zeros(B, 2 * H, 2 * W, cout + 16, dtype=torch.bfloat16, device=DEV), 8, cout) if up else None
    return Conv(Slice.full(x), wp, bp, cout, k, 1, k // 2, act, out=out, res=out if res else None, out2x=up2)


def test_widths_cover_every_instantiation():
    assert {instr_n(c) for c in COUTS} == {16, 32, 64, 96, 128, 160, 192, 224, 256}


@pytest.mark.parametrize("res", [False, True], ids=["plain", "residual"])
@pytest.mark.parametrize("act", [False, True], ids=["linear", "silu"])
@pytest.mark.parametrize("cout", COUTS)
def test_epilogue_every_width(cout, act, res):
    torch.manual_seed(cout)
    st = _stats()
    check_conv(make_conv(cout, 3 if cout <= 96 else 1, act, res, up=False), st, f"Cout {cout} (N {instr_n(cout)})")
    assert st["conv"] == 1 and st["bitwise"] == (0 if act else 1)


@pytest.mark.parametrize("cout,res", [(16, False), (32, True), (80, False), (128, True), (208, False), (320, True)])
def test_epilogue_upsampled_copy(cout, res):
    torch.manual_seed(cout + 1)
    st = _stats()
    check_conv(make_conv(cout, 1, False, res, up=True), st, f"Cout {cout} (N {instr_n(cout)}) with out2x")
    assert st["conv"] == 1 and st["bitwise"] == 1
