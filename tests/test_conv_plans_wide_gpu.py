"""Exact launch checks of the wide plans (yolov5l, yolov5x and the P6 models m6 / l6 / x6), and a census of the conv kernel
configurations every supported plan reaches.

The large models do not repeat the configurations of n / s / m at a larger size: Cout = 80 / 160 / 320 / 640 / 1280 (x) and
the 288 / 576 / 960 channel stages of the P6 family put the kernel at instruction N = 160 with 144 real columns, 80 real
columns in an N = 96 tile, 240 in an N = 256 tile, five N tiles per conv (Cout 1280, weights never resident), eight and ten
N tiles in the data gradients, and residual epilogues whose partial last 64-column block comes through cp.async.  Each
check below is test_conv_plans_exact_gpu's, imported rather than restated:

  1. every conv, records Detect, dgrad and wgrad launch of each plan against its own descriptor (check_conv /
     check_wgrad, integer operands, sentinels outside the write mask);
  2. the backward composition (dgrads equal conv2d_input of the forward weight, wgrads conv2d_weight) of yolov5x and of
     the four-level x6 graph;
  3. test_train_plans_pointwise_gpu's BatchNorm forward launches and backward steps of the yolov5x train plan;
  4. the census: a configuration key per conv launch, from the launch's descriptor and schedule alone (nothing is run);
     every key a supported plan reaches must be reached by a launch that some exact check runs.  A key only a plan
     reaches whose launches are not checked exactly gets a directed case: a small synthetic conv of that key.

Each case prints its launch counts, its runtime and its peak device memory (run with -s)."""
import math
import time

import pytest
import torch

from tests import test_conv_plans_exact_gpu as CE
from tests import test_train_plans_pointwise_gpu as TP
from tests.test_conv_epilogue_gpu import COUTS, make_conv
from tests.test_p6_gpu import _release_memory
from yolov5_obb_b200.conv import DETECT_GENERIC, MODE_DETECT, NO_PAIRW, Conv, Slice, pack_weights, tiling

pytestmark = pytest.mark.gpu
DEV = CE.DEV


def _measured(what, fn, *args):
    """fn(*args) with its wall time and peak device memory printed."""
    _release_memory()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    r = fn(*args)
    torch.cuda.synchronize()
    print(f"{what}: {time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB allocated")
    return r


# ---- 1. every launch of the wide plans against its descriptor --------------------------------------------------------
# the P6 plans at half the batch of the supported matrix; the census (4.) names what the full batch adds
WIDE = [
    ("l", 16, 1024, 1024, "forward"), ("l", 16, 1024, 1024, "records"), ("l", 8, 1024, 1024, "train"),
    ("x", 16, 1024, 1024, "forward"), ("x", 16, 1024, 1024, "records"), ("x", 8, 1024, 1024, "train"),
    ("m6", 8, 1280, 1280, "forward"), ("m6", 4, 1024, 1024, "train"),
    ("l6", 8, 1280, 1280, "forward"), ("l6", 4, 1024, 1024, "train"),
    ("x6", 8, 1280, 1280, "forward"), ("x6", 4, 1024, 1024, "train"),
]


def _id(size, B, H, W, kind):
    return f"yolov5{size}-b{B}-{H}x{W}-{kind}"


@pytest.mark.parametrize("size,B,H,W,kind", [pytest.param(*c, id=_id(*c)) for c in WIDE])
def test_every_launch_matches_its_descriptor(size, B, H, W, kind):
    _measured(_id(size, B, H, W, kind), CE.test_every_launch_matches_its_descriptor, size, B, H, W, kind)


# ---- 2. backward composition on the wide graphs ----------------------------------------------------------------------
@pytest.mark.parametrize("size,B,H,W", [pytest.param("x", 8, 1024, 1024, id="yolov5x-b8-1024"),
                                        pytest.param("x6", 8, 1024, 1024, id="yolov5x6-b8-1024")])
def test_backward_composition_exact(size, B, H, W):
    n_dgrad, n_acc, n_wgrad = _measured(f"yolov5{size} b{B} {H}x{W} composition", CE.backward_composition, size, B, H, W)
    assert n_dgrad > 0 and n_acc > 0 and n_wgrad > n_dgrad


# ---- 3. the pointwise launches of the yolov5x train plan -------------------------------------------------------------
def test_yolov5x_train_plan_forward_bn_launches():
    _measured("yolov5x b8 1024x1024 BatchNorm forward", TP.test_plan_forward_bn_launches, "x", 8, 1024, 1024)


def test_yolov5x_train_plan_backward_steps():
    _measured("yolov5x b8 1024x1024 backward steps", TP.test_plan_backward_steps, "x", 8, 1024, 1024)


# ---- 4. the census of conv configurations ----------------------------------------------------------------------------
KEY_FIELDS = ("inst", "N", "ragged", "multi_n", "resident", "ctas", "rowshift", "group", "KH", "stride", "pairw", "act",
              "out2x", "multi_tile")


def conv_key(op):
    """The kernel configuration of one Conv launch, from its descriptor and its schedule only (no pointer, no run):
    instantiation, instruction N, whether the last N tile has fewer real columns than N, more than one N tile, resident
    weights, CTAs per SM, row shift, units per stage, KH, stride, the pixel-pair view of stride-2 inputs, SiLU, the 2x copy,
    and whether some CTA runs more than one tile (ceil(B Hout Wout / 128) * n_tiles_n > grid, a sufficient condition)."""
    d, info = op.desc, op.info()
    detect = d.mode == MODE_DETECT
    _, bn, _, _, nt = tiling(d.Cin, d.Cout, d.mode, d.det_no)
    assert bn == info["block_n"]
    ni = 16 if bn <= 16 else (bn + 31) // 32 * 32
    last = d.det_no if detect else d.Cout - (nt - 1) * bn
    if detect:
        inst = "records" if (d.det_decode == 2 and d.det_no > 180 and ((d.det_no - 180 + 1) + 3) // 4 * 4 <= 64
                             and not d.flags & DETECT_GENERIC) else "detect"
    else:
        inst = "residual" if d.res else "plain"
    geom = d.out_h > 0
    hout = d.out_h if geom else (d.Hin + 2 * d.pad_h - d.KH) // d.stride + 1
    wout = d.out_w if geom else (d.Win + 2 * d.pad_w - d.KW) // d.stride + 1
    dense = d.in_row_stride in (0, d.in_pix_stride * d.Win)
    pairw = d.stride == 2 and d.Win % 2 == 0 and dense and not d.flags & NO_PAIRW
    multi = math.ceil(d.B * hout * wout / 128) * nt > info["grid"]
    return (inst, ni, last < ni, nt > 1, info["resident"], info["ctas_per_sm"], info["rowshift"], info["group"], d.KH,
            d.stride, int(pairw), d.act, int(bool(d.out2x)), int(multi))


def key_str(k):
    return " ".join(f"{f}={v}" for f, v in zip(KEY_FIELDS, k))


# {n, s, m, l, x} x {forward b16, records b16, train b8} at 1024^2; {n6 ... x6} x {forward b16 at 1280^2, train b8 at 1024^2}
SUPPORTED = [(s, 16, 1024, 1024, k) for s in "nsmlx" for k in ("forward", "records")] + \
            [(s, 8, 1024, 1024, "train") for s in "nsmlx"] + \
            [(s + "6", 16, 1280, 1280, "forward") for s in "nsmlx"] + [(s + "6", 8, 1024, 1024, "train") for s in "nsmlx"]
# the plans the exact launch checks run: test_conv_plans_exact_gpu's, test_p6_gpu's and this file's
CHECKED = [tuple(p.values) for p in CE.PLANS] + \
          [("s6", 16, 1280, 1280, "forward"), ("s6", 8, 1024, 1024, "train")] + WIDE
WIDE_SIZES = ("l", "x", "m6", "l6", "x6")


def _epilogue_convs():
    """test_conv_epilogue_gpu's convs."""
    convs = [make_conv(c, 3 if c <= 96 else 1, a, r, up=False) for c in COUTS for a in (False, True) for r in (False, True)]
    return convs + [make_conv(c, 1, False, r, up=True) for c, r in
                    [(16, False), (32, True), (80, False), (128, True), (208, False), (320, True)]]


# Directed cases: each reaches a key that a supported plan reaches and no checked plan does (the launch named), at a small
# shape: (cin, cout, (kh, kw), stride, act, residual, 2x copy, B, H, W).  The key depends on the channels, the kernel and
# the stride; the image size only decides the 2-CTA row shift (Wout >= 8), the pixel pairs (even Win) and whether a CTA
# runs several tiles: 2 x 128 x 144 outputs are 288 tiles, more than two CTAs on each of 132 SMs, 1 x 16 x 16 are two.
MT2, ONE = (2, 128, 144), (1, 16, 16)
MT2_S2 = (2, 256, 288)
DIRECTED = [
    # yolov5n b16 1024^2 forward: the stem (a 3 x 1 window of the space-to-depth input), 16 / 32 / 64 channels, many tiles
    (48, 16, (3, 1), 1, 1, 0, 0) + MT2,        # launch 0
    (16, 32, (3, 3), 2, 1, 0, 0) + MT2_S2,     # launch 1
    (16, 16, (1, 1), 1, 1, 0, 0) + MT2,        # launch 3
    (16, 16, (3, 3), 1, 1, 1, 0) + MT2,        # launch 4, Bottleneck
    (128, 64, (1, 1), 1, 1, 0, 1) + MT2,       # launch 34, with the 2x copy
    (32, 32, (3, 3), 1, 1, 0, 0) + MT2,        # launch 37
    (64, 64, (3, 3), 2, 1, 0, 0) + MT2_S2,     # launch 39
    # yolov5n b8 1024^2 train: the same without SiLU, and the data gradients (stride-2 phases: 2 x 1, 1 x 2, 2 x 2 taps)
    (48, 16, (3, 1), 1, 0, 0, 0) + MT2,        # launch 0
    (16, 32, (3, 3), 2, 0, 0, 0) + MT2_S2,     # launch 1
    (32, 16, (1, 1), 1, 0, 0, 0) + MT2,        # launch 2
    (16, 16, (3, 3), 1, 0, 0, 0) + MT2,        # launch 4
    (128, 128, (2, 1), 1, 0, 1, 0, 1, 32, 32),  # launch 70, accumulating
    (128, 128, (2, 2), 1, 0, 1, 0, 1, 32, 32),  # launch 71
    (64, 64, (2, 2), 1, 0, 1, 0, 2, 96, 96),   # launch 80: 2 x 97 x 97 outputs, 148 tiles on one CTA per SM
    (256, 128, (2, 2), 1, 0, 1, 0, 1, 32, 32),  # launch 103
    (16, 16, (1, 1), 1, 0, 1, 0) + MT2,        # launch 131
    (32, 16, (1, 2), 1, 0, 0, 0) + MT2,        # launch 134
    (32, 16, (2, 1), 1, 0, 0, 0) + MT2,        # launch 135
    (32, 16, (2, 2), 1, 0, 0, 0) + MT2,        # launch 136
    # yolov5n6 b16 1280^2 forward
    (96, 96, (1, 1), 1, 1, 0, 0) + ONE,        # launch 24
    (256, 192, (1, 1), 1, 1, 0, 1) + ONE,      # launch 34
    (256, 192, (1, 1), 1, 1, 0, 0, 2, 96, 96),  # launch 55: 144 tiles
    (192, 192, (3, 3), 2, 1, 0, 0, 1, 32, 32),  # launch 59
    # yolov5n6 b8 1024^2 train
    (192, 96, (1, 1), 1, 0, 0, 0) + ONE,       # launch 26
    (96, 96, (1, 1), 1, 0, 0, 0) + ONE,        # launch 27
    (96, 96, (3, 3), 1, 0, 0, 0) + ONE,        # launch 28
    (96, 96, (1, 1), 1, 0, 1, 0) + ONE,        # launch 142
    # the P6 plans at the supported batch: more tiles than the checked batch gives, so a CTA runs several of them
    (288, 576, (1, 1), 1, 0, 0, 0, 1, 64, 96),     # m6 b8 1024^2 train launch 182: 48 tiles x 3 N tiles on 132 CTAs
    (288, 576, (1, 1), 1, 0, 1, 0, 1, 64, 96),     # launch 187
    (1280, 960, (1, 1), 1, 1, 0, 1, 1, 64, 80),    # x6 b16 1280^2 forward launch 82: 40 tiles x 4 N tiles (240 in 256)
    (640, 960, (3, 3), 2, 0, 0, 0, 1, 128, 160),   # x6 b8 1024^2 train launch 61
]


def directed_conv(cin, cout, k, s, act, res, up, B, H, W):
    kh, kw = k
    g = torch.Generator(device="cpu").manual_seed(cin * 4096 + cout)
    w = torch.randn(cout, cin, kh, kw, generator=g).to(DEV)   # check_conv replaces weights, bias and activations by integers
    wp, bp = pack_weights(w, torch.randn(cout, generator=g).to(DEV))
    ho, wo = (H + 2 * (kh // 2) - kh) // s + 1, (W + 2 * (kw // 2) - kw) // s + 1
    x = torch.zeros(B, H, W, cin, dtype=torch.bfloat16, device=DEV)
    out = Slice(torch.zeros(B, ho, wo, cout + 16, dtype=torch.bfloat16, device=DEV), 8, cout)
    up2 = Slice(torch.zeros(B, 2 * ho, 2 * wo, cout + 16, dtype=torch.bfloat16, device=DEV), 8, cout) if up else None
    return Conv(Slice.full(x), wp, bp, cout, k, s, (kh // 2, kw // 2), act, out=out, res=out if res else None, out2x=up2)


def _directed_id(c):
    cin, cout, (kh, kw), s, act, res, up, B, H, W = c
    return f"{cin}-{cout}-k{kh}x{kw}s{s}" + ("-silu" if act else "") + ("-res" if res else "") + ("-up" if up else "") + \
        f"-b{B}-{H}x{W}"


@pytest.mark.parametrize("case", [pytest.param(c, id=_directed_id(c)) for c in DIRECTED])
def test_directed_case(case):
    torch.manual_seed(case[0] + case[1])
    st = CE._stats()
    CE.check_conv(directed_conv(*case), st, _directed_id(case))
    assert st["conv"] == 1 and st["bitwise"] == (0 if case[4] else 1)


def _plan_keys(plan, cache):
    """{key: its first launch} of one plan, built, read and freed (one plan at a time: the largest, yolov5x6 b16 at 1280^2,
    takes about 20 GiB)."""
    if plan in cache:
        return cache[plan]
    convs, _, keep = CE.plan_launches(*plan)
    keys = {}
    for i, op in enumerate(convs):
        d = op.desc
        keys.setdefault(conv_key(op), f"launch {i} (Cin {d.Cin} Cout {d.Cout} k{d.KH}x{d.KW} s{d.stride} "
                                      f"{d.B}x{d.Hin}x{d.Win} mode {d.mode} flags {d.flags})")
    del convs, keep
    _release_memory()
    cache[plan] = keys
    return keys


def census(checked=CHECKED, supported=SUPPORTED, directed=DIRECTED):
    """-> missing {key: (plan, launch)}: every key the supported plans reach that no checked plan, epilogue conv or
    directed case reaches.  Prints the key count per plan and the keys only the wide models reach."""
    cache = {}
    have = {}
    for plan in checked:
        for k in _plan_keys(plan, cache):
            have.setdefault(k, _id(*plan))
    for i, op in enumerate(_epilogue_convs()):
        have.setdefault(conv_key(op), f"epilogue conv {i}")
    for c in directed:
        have.setdefault(conv_key(directed_conv(*c)), f"directed {_directed_id(c)}")
    _release_memory()
    reached, missing = {}, {}
    print("\nconfiguration keys per supported plan:")
    for plan in supported:
        keys = _plan_keys(plan, cache)
        print(f"  {_id(*plan):32s} {len(keys):3d} keys")
        for k, i in keys.items():
            reached.setdefault(k, []).append((plan, i))
            if k not in have:
                missing.setdefault(k, (_id(*plan), i))
    only_wide = [k for k, by in reached.items() if all(p[0] in WIDE_SIZES for p, _ in by)]
    print(f"{len(reached)} keys over the supported plans, {len(have)} over the checked launches; "
          f"{len(only_wide)} reached only by {'/'.join(WIDE_SIZES)}:")
    for k in sorted(only_wide, key=str):
        print(f"  {key_str(k)}   ({', '.join(sorted({_id(*p) for p, _ in reached[k]}))})")
    for k, (plan, i) in missing.items():
        print(f"MISSING {key_str(k)}: {plan} {i}")
    return missing


def test_every_supported_configuration_is_checked():
    missing = _measured("census", census)
    assert not missing, f"{len(missing)} configurations of supported plans no exact check runs: " + \
        "; ".join(f"{key_str(k)} ({p} {i})" for k, (p, i) in missing.items())
