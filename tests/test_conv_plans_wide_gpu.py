"""Exact launch checks of the wide plans (yolov5l, yolov5x and the P6 models m6 / l6 / x6), and a census of the conv and
weight-gradient kernel configurations every supported plan reaches.

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
  4. the census: a configuration key per conv and per wgrad launch, from the launch's descriptor and schedule alone
     (nothing is run); every key a supported plan reaches must be reached by a launch that some exact check runs.  A key
     only a plan reaches whose launches are not checked exactly gets a directed case: a small synthetic conv or wgrad of
     that key.  "Supported" is every plan the entry points build at the sizes a user runs: forward, records and train at
     1024^2 (1280^2 for the P6 forward), whole-scene tiles, run_images' letterboxed and rectangular shapes, multi-scale
     train sizes, test-time augmentation and a frozen backbone.

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
from yolov5_obb_b200.train_ops import Wgrad

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


def _id(size, B, H, W, kind, freeze=None):
    return f"yolov5{size}-b{B}-{H}x{W}-{kind}" + (f"-freeze{freeze}" if freeze is not None else "")


@pytest.mark.parametrize("size,B,H,W,kind", [pytest.param(*c, id=_id(*c)) for c in WIDE])
def test_every_launch_matches_its_descriptor(size, B, H, W, kind):
    _measured(_id(size, B, H, W, kind), CE.test_every_launch_matches_its_descriptor, size, B, H, W, kind)


# the plan families beyond forward / records / train at the benchmarked sizes, each at a small size: a P6 records plan, both
# test-time-augmentation plans (de-scaled, de-flipped Detect rows), a non-square records plan (run_images' letterboxed and
# rectangular shapes), train plans whose P5 / P6 maps are odd (multi-scale sizes such as 544 or 576: no pixel pairs on the
# stride-2 convs that read them) and a train plan with a frozen backbone (--freeze 10: Concat gradients in channel windows)
FAMILIES = [
    ("n6", 2, 128, 192, "records", None), ("n", 2, 96, 160, "tta", None), ("n", 2, 96, 160, "tta-records", None),
    ("n", 1, 96, 320, "records", None), ("n", 2, 288, 288, "train", None), ("n6", 1, 192, 192, "train", None),
    ("s", 2, 128, 128, "train", 10),
    # the Detect launches a small plan does not reach: several tiles per CTA in every TTA branch, a records head whose P6
    # map (17 x 17 at 1088^2, SceneDetector's tiles) fits one tile per CTA
    ("s", 16, 1024, 1024, "tta", None), ("s", 16, 1024, 1024, "tta-records", None), ("s6", 16, 1088, 1088, "records", None),
]


@pytest.mark.parametrize("size,B,H,W,kind,freeze", [pytest.param(*c, id=_id(*c)) for c in FAMILIES])
def test_every_launch_of_the_plan_families_matches_its_descriptor(size, B, H, W, kind, freeze):
    _measured(_id(size, B, H, W, kind, freeze), CE.test_every_launch_matches_its_descriptor, size, B, H, W, kind, freeze)


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


# ---- 4. the census of conv and wgrad configurations ------------------------------------------------------------------
KEY_FIELDS = ("inst", "N", "ragged", "multi_n", "resident", "ctas", "rowshift", "group", "KH", "stride", "pairw", "act",
              "out2x", "multi_tile", "descale")


def conv_key(op):
    """The kernel configuration of one Conv launch, from its descriptor and its schedule only (no pointer, no run):
    instantiation, instruction N, whether the last N tile has fewer real columns than N, more than one N tile, resident
    weights, CTAs per SM, row shift, units per stage, KH, stride, the pixel-pair view of stride-2 inputs, SiLU, the 2x copy,
    whether some CTA runs more than one tile (ceil(B Hout Wout / 128) * n_tiles_n > grid, a sufficient condition), and the
    test-time-augmentation de-scale of the Detect epilogue (2: with the left-right de-flip)."""
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
    descale = (2 if d.det_flip_w > 0 else 1) if d.det_descale else 0
    return (inst, ni, last < ni, nt > 1, info["resident"], info["ctas_per_sm"], info["rowshift"], info["group"], d.KH,
            d.stride, int(pairw), d.act, int(bool(d.out2x)), int(multi), descale)


WGRAD_KEY_FIELDS = ("NC", "NC_last", "BN_ragged", "ci_short", "multi_ci", "multi_co", "co_last_le64", "co_ragged", "bk",
                    "w_ragged", "h_ragged", "ksplit", "ksplit_uneven", "ring_wraps", "stride", "taps", "x_strides",
                    "param_layout", "co_group")


def wgrad_key(wg):
    """The kernel configuration of one Wgrad launch, from its descriptor and the plan y5obb_wgrad_create chose (no pointer,
    no run): the consumer instantiations it reaches (NC = taps x b_chunks of the full tap groups, NC_last of a short last
    group, 0 when there is none), whether the CTA's input-channel block is narrower than its chunks (BN < 64 b_chunks) and
    whether the last ci block is short, more than one ci / co block, whether the last Cout block has at most 64 rows (one
    warpgroup) and whether Cout % 64 != 0, the pixel block size bk, whether the kwp x khp box leaves a partial block along Wo
    / Ho, split-K and an uneven split (steps % ksplit != 0), whether some CTA runs more steps than the pipeline has stages,
    the stride, KH x KW, the explicit x strides of the stem's window view, the parameter-layout dW strides and Detect's
    padded channel groups."""
    d, s = wg.desc, wg.info()
    ntaps = d.KH * d.KW
    last_taps = ntaps - (s["ngroups"] - 1) * s["T"]
    nc_last = last_taps * s["b_chunks"] if last_taps != s["T"] else 0
    co_last = d.Cout - (s["co_blks"] - 1) * 128
    return ("wgrad", min(4, s["T"] * s["b_chunks"]), min(4, nc_last), int(s["BN"] < 64 * s["b_chunks"]),
            int(d.Cin - (s["ci_blks"] - 1) * s["BN"] < s["BN"]), int(s["ci_blks"] > 1), int(s["co_blks"] > 1),
            int(co_last <= 64), int(d.Cout % 64 != 0), s["bk"], int(d.Wo % s["kwp"] != 0), int(d.Ho % s["khp"] != 0),
            int(s["ksplit"] > 1), int(s["steps"] % s["ksplit"] != 0), int(-(-s["steps"] // s["ksplit"]) > s["stages"]),
            d.stride, f"{d.KH}x{d.KW}", int(d.x_row_stride != 0), int(d.dw_tap_stride != 0), int(d.co_group_pad != 0))


def key_str(k):
    if k[0] == "wgrad":
        return "wgrad " + " ".join(f"{f}={v}" for f, v in zip(WGRAD_KEY_FIELDS, k[1:]))
    return "conv " + " ".join(f"{f}={v}" for f, v in zip(KEY_FIELDS, k))


# {n, s, m, l, x} x {forward b16, records b16, train b8} at 1024^2; {n6 ... x6} x {forward b16 at 1280^2, train b8 at 1024^2}
SUPPORTED = [(s, 16, 1024, 1024, k) for s in "nsmlx" for k in ("forward", "records")] + \
            [(s, 8, 1024, 1024, "train") for s in "nsmlx"] + \
            [(s + "6", 16, 1280, 1280, "forward") for s in "nsmlx"] + [(s + "6", 8, 1024, 1024, "train") for s in "nsmlx"]
BENCHMARKED = list(SUPPORTED)
# the plans the other entry points build
SUPPORTED += [(s + "6", 16, 1280, 1280, "records") for s in "nsmlx"]                       # detect_records on P6 models
SUPPORTED += [("s", 16, 1056, 1056, "records"), ("x", 16, 1056, 1056, "records"),         # SceneDetector tiles
              ("s6", 16, 1088, 1088, "records"), ("x6", 16, 1088, 1088, "records")]
SUPPORTED += [("s", 1, 1024, 576, "records"), ("s", 1, 320, 1024, "records"),             # run_images: letterboxed,
              ("s", 16, 768, 1024, "records")]                                            # rectangular batch shapes
SUPPORTED += [(s, 16, n, n, "train") for s in "sm" for n in (512, 544, 1504, 1536)] + \
             [("s6", 16, n, n, "train") for n in (576, 1536)]                              # train.py --multi-scale
SUPPORTED += [(s, 16, 1024, 1024, k) for s in "sm" for k in ("tta", "tta-records")]      # forward_augment, augment=True
SUPPORTED += [(s, 16, 1024, 1024, "train", 10) for s in "sm"]                             # train.py --freeze 10
# the plans the exact launch checks run: test_conv_plans_exact_gpu's, test_p6_gpu's and this file's
CHECKED = [tuple(p.values) for p in CE.PLANS] + \
          [("s6", 16, 1280, 1280, "forward"), ("s6", 8, 1024, 1024, "train")] + WIDE + FAMILIES
WIDE_SIZES = ("l", "x", "m6", "l6", "x6")


def _epilogue_convs():
    """test_conv_epilogue_gpu's convs."""
    convs = [make_conv(c, 3 if c <= 96 else 1, a, r, up=False) for c in COUTS for a in (False, True) for r in (False, True)]
    return convs + [make_conv(c, 1, False, r, up=True) for c, r in
                    [(16, False), (32, True), (80, False), (128, True), (208, False), (320, True)]]


# Directed cases: each reaches a key that a supported plan reaches and no checked plan does (the launch named), at a small
# shape: (cin, cout, (kh, kw), stride, act, residual, 2x copy, B, H, W[, the key it was added for]).  The key depends on the channels, the kernel and
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
    # train.py --multi-scale, m b16 at 1504^2: a 47 x 47 P5 map, two N tiles and several tiles per CTA
    (384, 384, (3, 3), 1, 0, 0, 0, 16, 47, 47,    # launch 40
     "conv inst=plain N=192 ragged=False multi_n=True resident=0 ctas=1 rowshift=0 group=1 KH=3 stride=1 pairw=0 act=0 "
     "out2x=0 multi_tile=1 descale=0"),
    (384, 384, (2, 1), 1, 0, 1, 0, 16, 47, 47,    # launch 94, a stride-2 data-gradient phase, accumulating
     "conv inst=residual N=192 ragged=False multi_n=True resident=0 ctas=1 rowshift=0 group=1 KH=2 stride=1 pairw=0 act=0 "
     "out2x=0 multi_tile=1 descale=0"),
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
    cin, cout, (kh, kw), s, act, res, up, B, H, W = c[:10]
    return f"{cin}-{cout}-k{kh}x{kw}s{s}" + ("-silu" if act else "") + ("-res" if res else "") + ("-up" if up else "") + \
        f"-b{B}-{H}x{W}"


@pytest.mark.parametrize("case", [pytest.param(c, id=_directed_id(c)) for c in DIRECTED])
def test_directed_case(case):
    torch.manual_seed(case[0] + case[1])
    op = directed_conv(*case[:10])
    if len(case) > 10:   # the key the case was added for, which the SM count may move
        assert key_str(conv_key(op)) == case[10], f"the case reaches {key_str(conv_key(op))}, not {case[10]}"
    st = CE._stats()
    CE.check_conv(op, st, _directed_id(case))
    assert st["conv"] == 1 and st["bitwise"] == (0 if case[4] else 1)


# Directed wgrad cases: each reaches a wgrad key that a supported plan reaches and no checked plan does (the launch named),
# with the key it was added for: (cin, cout, (kh, kw), stride, B, H, W, form, key: the values of WGRAD_KEY_FIELDS).  Each
# is the launch named at a batch (1, 2, 4, 8 or the plan's) that still reaches the key.  form "conv": a Conv layer's weight
# gradient in the parameter layout; "detect": Detect's, 1x1 over padded channel groups (cout = 3 groups of 208 of which
# 200 are real); "stem": the stem's 3x1 window view of the space-to-depth image (cin 48).  ksplit and the grid follow
# the SM count, so each case asserts on the device it runs on that it still reaches its key.
DIRECTED_WGRAD = [
    # yolov5n-b8-1024x1024-train wgrad 0
    (64, 624, (1, 1), 1, 1, 128, 128, 'detect', (1, 0, 0, 0, 0, 1, 0, 1, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 1)),
    # yolov5n-b8-1024x1024-train wgrad 10
    (128, 64, (1, 1), 1, 1, 64, 64, 'conv', (2, 0, 0, 0, 0, 0, 1, 0, 128, 0, 0, 1, 0, 0, 1, '1x1', 0, 1, 0)),
    # yolov5n-b8-1024x1024-train wgrad 14
    (64, 64, (3, 3), 2, 8, 128, 128, 'conv', (3, 0, 0, 0, 0, 0, 1, 0, 128, 0, 0, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5n-b8-1024x1024-train wgrad 16
    (128, 32, (1, 1), 1, 8, 128, 128, 'conv', (2, 0, 0, 0, 0, 0, 1, 1, 128, 0, 0, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5n-b8-1024x1024-train wgrad 58
    (16, 32, (3, 3), 2, 1, 512, 512, 'conv', (3, 0, 1, 0, 0, 0, 1, 1, 128, 0, 0, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5n6-b8-1024x1024-train wgrad 3
    (256, 624, (1, 1), 1, 2, 16, 16, 'detect', (4, 0, 0, 0, 0, 1, 0, 1, 128, 0, 0, 1, 0, 0, 1, '1x1', 0, 1, 1)),
    # yolov5n6-b8-1024x1024-train wgrad 5
    (384, 128, (1, 1), 1, 2, 16, 16, 'conv', (3, 0, 0, 0, 1, 0, 0, 0, 128, 0, 0, 1, 0, 0, 1, '1x1', 0, 1, 0)),
    # yolov5n6-b8-1024x1024-train wgrad 6
    (128, 128, (3, 3), 1, 2, 16, 16, 'conv', (4, 2, 0, 0, 0, 0, 0, 0, 128, 0, 0, 1, 0, 0, 1, '3x3', 0, 1, 0)),
    # yolov5n6-b8-1024x1024-train wgrad 11
    (256, 96, (1, 1), 1, 1, 32, 32, 'conv', (4, 0, 0, 0, 0, 0, 0, 1, 128, 0, 0, 1, 0, 0, 1, '1x1', 0, 1, 0)),
    # yolov5n6-b8-1024x1024-train wgrad 13
    (96, 96, (1, 1), 1, 1, 32, 32, 'conv', (2, 0, 1, 0, 0, 0, 0, 1, 128, 0, 0, 1, 0, 0, 1, '1x1', 0, 1, 0)),
    # yolov5n6-b8-1024x1024-train wgrad 33
    (192, 128, (1, 1), 1, 1, 32, 32, 'conv', (3, 0, 0, 0, 0, 0, 0, 0, 128, 0, 0, 1, 0, 0, 1, '1x1', 0, 1, 0)),
    # yolov5n6-b8-1024x1024-train wgrad 35
    (384, 96, (1, 1), 1, 1, 32, 32, 'conv', (3, 0, 0, 0, 1, 0, 0, 1, 128, 0, 0, 1, 0, 0, 1, '1x1', 0, 1, 0)),
    # yolov5n6-b8-1024x1024-train wgrad 39
    (256, 192, (1, 1), 1, 2, 16, 16, 'conv', (4, 0, 0, 0, 0, 1, 1, 0, 128, 0, 0, 1, 0, 0, 1, '1x1', 0, 1, 0)),
    # yolov5n6-b8-1024x1024-train wgrad 49
    (192, 96, (1, 1), 1, 1, 32, 32, 'conv', (3, 0, 0, 0, 0, 0, 0, 1, 128, 0, 0, 1, 0, 0, 1, '1x1', 0, 1, 0)),
    # yolov5n6-b8-1024x1024-train wgrad 53
    (128, 192, (3, 3), 2, 4, 64, 64, 'conv', (4, 2, 0, 0, 0, 1, 1, 0, 128, 0, 0, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5m6-b8-1024x1024-train wgrad 11
    (576, 576, (3, 3), 2, 8, 32, 32, 'conv', (3, 0, 0, 0, 1, 1, 1, 0, 128, 0, 0, 1, 0, 1, 2, '3x3', 0, 1, 0)),
    # yolov5m6-b8-1024x1024-train wgrad 15
    (288, 288, (1, 1), 1, 8, 32, 32, 'conv', (3, 0, 1, 0, 1, 1, 1, 1, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5x6-b8-1024x1024-train wgrad 101
    (640, 960, (3, 3), 2, 8, 64, 64, 'conv', (4, 0, 1, 1, 1, 1, 1, 0, 128, 0, 0, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5s-b16-512x512-train wgrad 22
    (512, 128, (1, 1), 1, 1, 32, 32, 'conv', (4, 0, 0, 0, 1, 0, 0, 0, 128, 0, 0, 1, 0, 0, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 0
    (128, 624, (1, 1), 1, 2, 68, 68, 'detect', (2, 0, 0, 0, 0, 1, 0, 1, 128, 1, 1, 1, 1, 1, 1, '1x1', 0, 1, 1)),
    # yolov5s-b16-544x544-train wgrad 1
    (256, 624, (1, 1), 1, 4, 34, 34, 'detect', (4, 0, 0, 0, 0, 1, 0, 1, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 1)),
    # yolov5s-b16-544x544-train wgrad 2
    (512, 624, (1, 1), 1, 16, 17, 17, 'detect', (4, 0, 0, 0, 1, 1, 0, 1, 128, 1, 1, 1, 1, 1, 1, '1x1', 0, 1, 1)),
    # yolov5s-b16-544x544-train wgrad 3
    (512, 512, (1, 1), 1, 16, 17, 17, 'conv', (4, 0, 0, 0, 1, 1, 0, 0, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 4
    (512, 256, (1, 1), 1, 16, 17, 17, 'conv', (4, 0, 0, 0, 1, 1, 0, 0, 128, 1, 1, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 5
    (256, 256, (3, 3), 1, 4, 17, 17, 'conv', (4, 0, 0, 0, 0, 1, 0, 0, 128, 1, 1, 1, 1, 1, 1, '3x3', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 6
    (256, 256, (1, 1), 1, 2, 17, 17, 'conv', (4, 0, 0, 0, 0, 1, 0, 0, 128, 1, 1, 1, 0, 0, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 8
    (256, 256, (3, 3), 2, 4, 34, 34, 'conv', (4, 0, 0, 0, 0, 1, 0, 0, 128, 1, 1, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 9
    (256, 256, (1, 1), 1, 16, 34, 34, 'conv', (4, 0, 0, 0, 0, 1, 0, 0, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 10
    (256, 128, (1, 1), 1, 1, 34, 34, 'conv', (4, 0, 0, 0, 0, 0, 0, 0, 128, 1, 1, 1, 0, 0, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 11
    (128, 128, (3, 3), 1, 4, 34, 34, 'conv', (4, 2, 0, 0, 0, 0, 0, 0, 128, 1, 1, 1, 0, 1, 1, '3x3', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 14
    (128, 128, (3, 3), 2, 4, 68, 68, 'conv', (4, 2, 0, 0, 0, 0, 0, 0, 128, 1, 1, 1, 0, 1, 2, '3x3', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 15
    (128, 128, (1, 1), 1, 16, 68, 68, 'conv', (2, 0, 0, 0, 0, 0, 0, 0, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 16
    (256, 64, (1, 1), 1, 8, 68, 68, 'conv', (4, 0, 0, 0, 0, 0, 1, 0, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 17
    (64, 64, (3, 3), 1, 16, 68, 68, 'conv', (3, 0, 0, 0, 0, 0, 1, 0, 128, 1, 1, 1, 1, 1, 1, '3x3', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 22
    (512, 128, (1, 1), 1, 16, 34, 34, 'conv', (4, 0, 0, 0, 1, 0, 0, 0, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 44
    (128, 256, (3, 3), 2, 16, 68, 68, 'conv', (4, 2, 0, 0, 0, 1, 0, 0, 128, 1, 1, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 46
    (128, 64, (1, 1), 1, 16, 68, 68, 'conv', (2, 0, 0, 0, 0, 0, 1, 0, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 52
    (64, 128, (3, 3), 2, 16, 136, 136, 'conv', (3, 0, 0, 0, 0, 0, 0, 0, 128, 1, 1, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 53
    (64, 64, (1, 1), 1, 8, 136, 136, 'conv', (1, 0, 0, 0, 0, 0, 1, 0, 128, 1, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 54
    (64, 32, (1, 1), 1, 8, 136, 136, 'conv', (1, 0, 0, 0, 0, 0, 1, 1, 128, 1, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 55
    (32, 32, (3, 3), 1, 1, 136, 136, 'conv', (3, 0, 1, 0, 0, 0, 1, 1, 128, 1, 0, 1, 1, 1, 1, '3x3', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 56
    (32, 32, (1, 1), 1, 8, 136, 136, 'conv', (1, 0, 1, 0, 0, 0, 1, 1, 128, 1, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-544x544-train wgrad 58
    (32, 64, (3, 3), 2, 1, 272, 272, 'conv', (3, 0, 1, 0, 0, 0, 1, 0, 128, 1, 0, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5s-b16-1504x1504-train wgrad 0
    (128, 624, (1, 1), 1, 1, 188, 188, 'detect', (2, 0, 0, 0, 0, 1, 0, 1, 128, 1, 0, 1, 1, 1, 1, '1x1', 0, 1, 1)),
    # yolov5s-b16-1504x1504-train wgrad 1
    (256, 624, (1, 1), 1, 8, 94, 94, 'detect', (4, 0, 0, 0, 0, 1, 0, 1, 128, 1, 1, 1, 1, 1, 1, '1x1', 0, 1, 1)),
    # yolov5s-b16-1504x1504-train wgrad 6
    (256, 256, (1, 1), 1, 16, 47, 47, 'conv', (4, 0, 0, 0, 0, 1, 0, 0, 128, 1, 1, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-1504x1504-train wgrad 10
    (256, 128, (1, 1), 1, 4, 94, 94, 'conv', (4, 0, 0, 0, 0, 0, 0, 0, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-1504x1504-train wgrad 11
    (128, 128, (3, 3), 1, 8, 94, 94, 'conv', (4, 2, 0, 0, 0, 0, 0, 0, 128, 1, 1, 1, 1, 1, 1, '3x3', 0, 1, 0)),
    # yolov5s-b16-1504x1504-train wgrad 14
    (128, 128, (3, 3), 2, 8, 188, 188, 'conv', (4, 2, 0, 0, 0, 0, 0, 0, 128, 1, 1, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5s-b16-1504x1504-train wgrad 15
    (128, 128, (1, 1), 1, 2, 188, 188, 'conv', (2, 0, 0, 0, 0, 0, 0, 0, 128, 1, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-1504x1504-train wgrad 16
    (256, 64, (1, 1), 1, 2, 188, 188, 'conv', (4, 0, 0, 0, 0, 0, 1, 0, 128, 1, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-1504x1504-train wgrad 17
    (64, 64, (3, 3), 1, 1, 188, 188, 'conv', (3, 0, 0, 0, 0, 0, 1, 0, 128, 1, 0, 1, 1, 1, 1, '3x3', 0, 1, 0)),
    # yolov5s-b16-1504x1504-train wgrad 46
    (128, 64, (1, 1), 1, 2, 188, 188, 'conv', (2, 0, 0, 0, 0, 0, 1, 0, 128, 1, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-1504x1504-train wgrad 52
    (64, 128, (3, 3), 2, 1, 376, 376, 'conv', (3, 0, 0, 0, 0, 0, 0, 0, 128, 1, 0, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5s-b16-1536x1536-train wgrad 6
    (256, 256, (1, 1), 1, 16, 48, 48, 'conv', (4, 0, 0, 0, 0, 1, 0, 0, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-1536x1536-train wgrad 15
    (128, 128, (1, 1), 1, 2, 192, 192, 'conv', (2, 0, 0, 0, 0, 0, 0, 0, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-1536x1536-train wgrad 16
    (256, 64, (1, 1), 1, 2, 192, 192, 'conv', (4, 0, 0, 0, 0, 0, 1, 0, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-1536x1536-train wgrad 18
    (64, 64, (1, 1), 1, 16, 192, 192, 'conv', (1, 0, 0, 0, 0, 0, 1, 0, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-1536x1536-train wgrad 46
    (128, 64, (1, 1), 1, 2, 192, 192, 'conv', (2, 0, 0, 0, 0, 0, 1, 0, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-1536x1536-train wgrad 54
    (64, 32, (1, 1), 1, 4, 384, 384, 'conv', (1, 0, 0, 0, 0, 0, 1, 1, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s-b16-1536x1536-train wgrad 56
    (32, 32, (1, 1), 1, 4, 384, 384, 'conv', (1, 0, 1, 0, 0, 0, 1, 1, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 0
    (192, 624, (1, 1), 1, 2, 68, 68, 'detect', (3, 0, 0, 0, 0, 1, 0, 1, 128, 1, 1, 1, 1, 1, 1, '1x1', 0, 1, 1)),
    # yolov5m-b16-544x544-train wgrad 1
    (384, 624, (1, 1), 1, 16, 34, 34, 'detect', (3, 0, 0, 0, 1, 1, 0, 1, 128, 1, 1, 1, 1, 1, 1, '1x1', 0, 1, 1)),
    # yolov5m-b16-544x544-train wgrad 2
    (768, 624, (1, 1), 1, 8, 17, 17, 'detect', (4, 0, 0, 0, 1, 1, 0, 1, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 1)),
    # yolov5m-b16-544x544-train wgrad 5
    (384, 384, (3, 3), 1, 2, 17, 17, 'conv', (3, 0, 0, 0, 1, 1, 0, 0, 128, 1, 1, 1, 0, 1, 1, '3x3', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 6
    (384, 384, (1, 1), 1, 16, 17, 17, 'conv', (3, 0, 0, 0, 1, 1, 0, 0, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 10
    (384, 384, (3, 3), 2, 2, 34, 34, 'conv', (3, 0, 0, 0, 1, 1, 0, 0, 128, 1, 1, 1, 0, 1, 2, '3x3', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 11
    (384, 384, (1, 1), 1, 16, 34, 34, 'conv', (3, 0, 0, 0, 1, 1, 0, 0, 128, 1, 1, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 12
    (384, 192, (1, 1), 1, 8, 34, 34, 'conv', (3, 0, 0, 0, 1, 1, 1, 0, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 13
    (192, 192, (3, 3), 1, 4, 34, 34, 'conv', (3, 0, 0, 0, 0, 1, 1, 0, 128, 1, 1, 1, 1, 1, 1, '3x3', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 14
    (192, 192, (1, 1), 1, 16, 34, 34, 'conv', (3, 0, 0, 0, 0, 1, 1, 0, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 18
    (192, 192, (3, 3), 2, 4, 68, 68, 'conv', (3, 0, 0, 0, 0, 1, 1, 0, 128, 1, 1, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 19
    (192, 192, (1, 1), 1, 16, 68, 68, 'conv', (3, 0, 0, 0, 0, 1, 1, 0, 128, 1, 1, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 20
    (384, 96, (1, 1), 1, 16, 68, 68, 'conv', (3, 0, 0, 0, 1, 0, 0, 1, 128, 1, 1, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 21
    (96, 96, (3, 3), 1, 2, 68, 68, 'conv', (4, 2, 1, 0, 0, 0, 0, 1, 128, 1, 1, 1, 1, 1, 1, '3x3', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 22
    (96, 96, (1, 1), 1, 16, 68, 68, 'conv', (2, 0, 1, 0, 0, 0, 0, 1, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 28
    (768, 192, (1, 1), 1, 16, 34, 34, 'conv', (4, 0, 0, 0, 1, 1, 1, 0, 128, 1, 1, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 44
    (384, 768, (3, 3), 2, 2, 34, 34, 'conv', (3, 0, 0, 0, 1, 1, 0, 0, 128, 1, 1, 0, 0, 1, 2, '3x3', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 60
    (192, 384, (3, 3), 2, 1, 68, 68, 'conv', (3, 0, 0, 0, 0, 1, 0, 0, 128, 1, 1, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 62
    (192, 96, (1, 1), 1, 8, 68, 68, 'conv', (3, 0, 0, 0, 0, 0, 0, 1, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 72
    (96, 192, (3, 3), 2, 1, 136, 136, 'conv', (4, 2, 1, 0, 0, 1, 1, 0, 128, 1, 1, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 73
    (96, 96, (1, 1), 1, 4, 136, 136, 'conv', (2, 0, 1, 0, 0, 0, 0, 1, 128, 1, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 74
    (96, 48, (1, 1), 1, 4, 136, 136, 'conv', (2, 0, 1, 0, 0, 0, 1, 1, 128, 1, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-544x544-train wgrad 80
    (48, 96, (3, 3), 2, 1, 272, 272, 'conv', (3, 0, 1, 0, 0, 0, 0, 1, 128, 1, 0, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5m-b16-1504x1504-train wgrad 0
    (192, 624, (1, 1), 1, 1, 188, 188, 'detect', (3, 0, 0, 0, 0, 1, 0, 1, 128, 1, 0, 1, 1, 1, 1, '1x1', 0, 1, 1)),
    # yolov5m-b16-1504x1504-train wgrad 5
    (384, 384, (3, 3), 1, 8, 47, 47, 'conv', (3, 0, 0, 0, 1, 1, 0, 0, 128, 1, 1, 1, 1, 1, 1, '3x3', 0, 1, 0)),
    # yolov5m-b16-1504x1504-train wgrad 10
    (384, 384, (3, 3), 2, 8, 94, 94, 'conv', (3, 0, 0, 0, 1, 1, 0, 0, 128, 1, 1, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5m-b16-1504x1504-train wgrad 12
    (384, 192, (1, 1), 1, 2, 94, 94, 'conv', (3, 0, 0, 0, 1, 1, 1, 0, 128, 1, 1, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-1504x1504-train wgrad 19
    (192, 192, (1, 1), 1, 1, 188, 188, 'conv', (3, 0, 0, 0, 0, 1, 1, 0, 128, 1, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-1504x1504-train wgrad 20
    (384, 96, (1, 1), 1, 1, 188, 188, 'conv', (3, 0, 0, 0, 1, 0, 0, 1, 128, 1, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-1504x1504-train wgrad 21
    (96, 96, (3, 3), 1, 1, 188, 188, 'conv', (4, 2, 1, 0, 0, 0, 0, 1, 128, 1, 0, 1, 1, 1, 1, '3x3', 0, 1, 0)),
    # yolov5m-b16-1504x1504-train wgrad 62
    (192, 96, (1, 1), 1, 2, 188, 188, 'conv', (3, 0, 0, 0, 0, 0, 0, 1, 128, 1, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-1504x1504-train wgrad 72
    (96, 192, (3, 3), 2, 1, 376, 376, 'conv', (4, 2, 1, 0, 0, 1, 1, 0, 128, 1, 0, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5m-b16-1536x1536-train wgrad 5
    (384, 384, (3, 3), 1, 8, 48, 48, 'conv', (3, 0, 0, 0, 1, 1, 0, 0, 128, 0, 0, 1, 1, 1, 1, '3x3', 0, 1, 0)),
    # yolov5m-b16-1536x1536-train wgrad 10
    (384, 384, (3, 3), 2, 8, 96, 96, 'conv', (3, 0, 0, 0, 1, 1, 0, 0, 128, 0, 0, 1, 1, 1, 2, '3x3', 0, 1, 0)),
    # yolov5m-b16-1536x1536-train wgrad 12
    (384, 192, (1, 1), 1, 2, 96, 96, 'conv', (3, 0, 0, 0, 1, 1, 1, 0, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-1536x1536-train wgrad 19
    (192, 192, (1, 1), 1, 1, 192, 192, 'conv', (3, 0, 0, 0, 0, 1, 1, 0, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-1536x1536-train wgrad 20
    (384, 96, (1, 1), 1, 1, 192, 192, 'conv', (3, 0, 0, 0, 1, 0, 0, 1, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-1536x1536-train wgrad 22
    (96, 96, (1, 1), 1, 2, 192, 192, 'conv', (2, 0, 1, 0, 0, 0, 0, 1, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-1536x1536-train wgrad 62
    (192, 96, (1, 1), 1, 2, 192, 192, 'conv', (3, 0, 0, 0, 0, 0, 0, 1, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5m-b16-1536x1536-train wgrad 74
    (96, 48, (1, 1), 1, 4, 384, 384, 'conv', (2, 0, 1, 0, 0, 0, 1, 1, 128, 0, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s6-b16-576x576-train wgrad 4
    (512, 512, (1, 1), 1, 8, 9, 9, 'conv', (4, 0, 0, 0, 1, 1, 0, 0, 128, 1, 1, 1, 0, 0, 1, '1x1', 0, 1, 0)),
    # yolov5s6-b16-576x576-train wgrad 13
    (192, 192, (1, 1), 1, 2, 18, 18, 'conv', (3, 0, 0, 0, 0, 1, 1, 0, 128, 1, 1, 1, 0, 0, 1, '1x1', 0, 1, 0)),
    # yolov5s6-b16-576x576-train wgrad 22
    (128, 128, (1, 1), 1, 16, 72, 72, 'conv', (2, 0, 0, 0, 0, 0, 0, 0, 128, 1, 0, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s6-b16-576x576-train wgrad 23
    (256, 64, (1, 1), 1, 8, 72, 72, 'conv', (4, 0, 0, 0, 0, 0, 1, 0, 128, 1, 0, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s6-b16-576x576-train wgrad 35
    (768, 192, (1, 1), 1, 16, 18, 18, 'conv', (4, 0, 0, 0, 1, 1, 1, 0, 128, 1, 1, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s6-b16-576x576-train wgrad 53
    (256, 384, (3, 3), 2, 4, 36, 36, 'conv', (4, 0, 0, 0, 0, 1, 0, 0, 128, 1, 1, 1, 0, 1, 2, '3x3', 0, 1, 0)),
    # yolov5s6-b16-576x576-train wgrad 65
    (128, 64, (1, 1), 1, 16, 72, 72, 'conv', (2, 0, 0, 0, 0, 0, 1, 0, 128, 1, 0, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s6-b16-1536x1536-train wgrad 3
    (512, 624, (1, 1), 1, 8, 24, 24, 'detect', (4, 0, 0, 0, 1, 1, 0, 1, 128, 1, 0, 1, 0, 1, 1, '1x1', 0, 1, 1)),
    # yolov5s6-b16-1536x1536-train wgrad 4
    (512, 512, (1, 1), 1, 8, 24, 24, 'conv', (4, 0, 0, 0, 1, 1, 0, 0, 128, 1, 0, 1, 0, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s6-b16-1536x1536-train wgrad 5
    (768, 256, (1, 1), 1, 16, 24, 24, 'conv', (4, 0, 0, 0, 1, 1, 0, 0, 128, 1, 0, 1, 1, 1, 1, '1x1', 0, 1, 0)),
    # yolov5s6-b16-1536x1536-train wgrad 6
    (256, 256, (3, 3), 1, 8, 24, 24, 'conv', (4, 0, 0, 0, 0, 1, 0, 0, 128, 1, 0, 1, 1, 1, 1, '3x3', 0, 1, 0)),
    # yolov5s6-b16-1536x1536-train wgrad 7
    (256, 256, (1, 1), 1, 1, 24, 24, 'conv', (4, 0, 0, 0, 0, 1, 0, 0, 128, 1, 0, 1, 0, 0, 1, '1x1', 0, 1, 0)),
    # yolov5s6-b16-1536x1536-train wgrad 9
    (384, 384, (3, 3), 2, 1, 48, 48, 'conv', (3, 0, 0, 0, 1, 1, 0, 0, 128, 1, 0, 1, 0, 1, 2, '3x3', 0, 1, 0)),
    # yolov5s6-b16-1536x1536-train wgrad 33
    (384, 256, (1, 1), 1, 4, 48, 48, 'conv', (3, 0, 0, 0, 1, 1, 0, 0, 128, 0, 0, 1, 0, 1, 1, '1x1', 0, 1, 0)),
]


def directed_wgrad(cin, cout, k, s, B, H, W, form="conv"):
    kh, kw = k
    g = torch.Generator(device="cpu").manual_seed(cin * 4096 + cout)
    if form == "stem":       # x_s2d [B, H, W + 2, 16]: 48-channel windows at a 16-channel pixel stride
        x = torch.randn(B, H, W + 2, 16, generator=g).to(DEV).bfloat16()
        dz = torch.zeros(B, H, W, cout, dtype=torch.bfloat16, device=DEV)
        dw = torch.zeros(3 * cout * 48, device=DEV)
        return Wgrad(dz.data_ptr(), cout, x.data_ptr(), 16, dw, B, cout, H, W, 48, H, W, (3, 1), 1, (1, 0), keep=(dz, x),
                     x_strides=((W + 2) * 16, H * (W + 2) * 16))
    ph, pw = kh // 2, kw // 2
    ho, wo = (H + 2 * ph - kh) // s + 1, (W + 2 * pw - kw) // s + 1
    x = torch.zeros(B, H, W, cin + 16, dtype=torch.bfloat16, device=DEV)      # channel slices [8, 8 + C) of wider buffers
    dz = torch.zeros(B, ho, wo, cout + 16, dtype=torch.bfloat16, device=DEV)
    if form == "detect":
        assert k == (1, 1) and s == 1 and cout % 208 == 0
        dw = torch.zeros(cout // 208 * 200, cin, 1, 1, device=DEV)
        return Wgrad(dz.data_ptr() + 16, cout + 16, x.data_ptr() + 16, cin + 16, dw, B, cout, ho, wo, cin, H, W, 1, 1, 0,
                     keep=(dz, x), param_layout=True, co_group=(200, 208))
    dw = torch.zeros(cout, cin, kh, kw, device=DEV)
    return Wgrad(dz.data_ptr() + 16, cout + 16, x.data_ptr() + 16, cin + 16, dw, B, cout, ho, wo, cin, H, W, k, s, (ph, pw),
                 keep=(dz, x), param_layout=True)


def _directed_wgrad_id(c):
    cin, cout, (kh, kw), s, B, H, W, form = c[:8]
    return f"{form}-{cin}-{cout}-k{kh}x{kw}s{s}-b{B}-{H}x{W}"


@pytest.mark.parametrize("case", [pytest.param(c, id=_directed_wgrad_id(c)) for c in DIRECTED_WGRAD])
def test_directed_wgrad_case(case):
    torch.manual_seed(case[0] + case[1])
    wg = directed_wgrad(*case[:8])
    want = ("wgrad",) + tuple(case[8])
    assert wgrad_key(wg) == want, f"on this device ({torch.cuda.get_device_properties(0).multi_processor_count} SMs) the " \
                                  f"case reaches {key_str(wgrad_key(wg))}, not the key it was added for: {key_str(want)}"
    st = CE._stats()
    CE.check_wgrad(wg, st, _directed_wgrad_id(case))
    assert st["wgrad"] == 1


def _launch_str(i, d, what):
    if what == "wgrad":
        return f"wgrad {i} (Cin {d.Cin} Cout {d.Cout} k{d.KH}x{d.KW} s{d.stride} {d.B}x{d.Ho}x{d.Wo} " \
               f"co_group {d.co_group}/{d.co_group_pad} x_row_stride {d.x_row_stride})"
    return f"launch {i} (Cin {d.Cin} Cout {d.Cout} k{d.KH}x{d.KW} s{d.stride} {d.B}x{d.Hin}x{d.Win} mode {d.mode} " \
           f"flags {d.flags} descale {d.det_descale})"


def plan_keys(plan):
    """{key: its first launch} of one plan (conv and wgrad keys).  A train plan is built with AliasCarver: its buffers
    alias one allocation, so the largest (m b16 at 1536^2) is keyed at the batch train.py runs without its activations;
    test_alias_built_plans_key_like_allocated_ones shows that this changes no key."""
    size, B, H, W, kind = plan[:5]
    freeze = plan[5] if len(plan) > 5 else None
    convs, wgrads, keep = CE.plan_launches(size, B, H, W, kind, freeze, key_only=kind == "train")
    keys = {}
    for i, op in enumerate(convs):
        keys.setdefault(conv_key(op), _launch_str(i, op.desc, "conv"))
    for i, wg in enumerate(wgrads):
        keys.setdefault(wgrad_key(wg), _launch_str(i, wg.desc, "wgrad"))
    del convs, wgrads, keep
    _release_memory()
    return keys


def _plan_keys(plan, cache):
    """plan_keys, built, read and freed once per plan (one plan at a time: the largest, yolov5x6 b16 at 1280^2, takes
    about 20 GiB)."""
    if plan not in cache:
        cache[plan] = plan_keys(plan)
    return cache[plan]


def test_alias_built_plans_key_like_allocated_ones():
    """The census keys train plans built on aliased buffers: their launches, conv and wgrad, key exactly as those of the
    same plan on its own buffers (keys depend on shapes, strides and schedules, never on addresses)."""
    for plan in [("n", 2, 96, 160), ("s", 2, 128, 128)]:
        for freeze in (None, 10):
            got = []
            for key_only in (False, True):
                convs, wgrads, keep = CE.plan_launches(*plan, "train", freeze, key_only=key_only)
                got.append([conv_key(op) for op in convs] + [wgrad_key(wg) for wg in wgrads])
                del convs, wgrads, keep
                _release_memory()
            assert got[0] == got[1], (plan, freeze)


def census(checked=CHECKED, supported=SUPPORTED, directed=DIRECTED, directed_wgrad_cases=DIRECTED_WGRAD):
    """-> missing {key: (plan, launch)}: every conv or wgrad key the supported plans reach that no checked plan, epilogue
    conv or directed case reaches.  Prints the conv and wgrad key counts per plan, the keys only the wide models reach and
    the keys only the entry-point plans beyond the benchmarked ones reach."""
    cache = {}
    have = {}
    for plan in checked:
        for k in _plan_keys(plan, cache):
            have.setdefault(k, _id(*plan))
    for i, op in enumerate(_epilogue_convs()):
        have.setdefault(conv_key(op), f"epilogue conv {i}")
    for c in directed:
        have.setdefault(conv_key(directed_conv(*c[:10])), f"directed {_directed_id(c)}")
    for c in directed_wgrad_cases:
        have.setdefault(wgrad_key(directed_wgrad(*c[:8])), f"directed wgrad {_directed_wgrad_id(c)}")
    _release_memory()
    reached, missing = {}, {}
    print("\nconfiguration keys per supported plan (conv, wgrad):")
    for plan in supported:
        keys = _plan_keys(plan, cache)
        nw = sum(1 for k in keys if k[0] == "wgrad")
        print(f"  {_id(*plan):40s} {len(keys) - nw:3d} conv {nw:3d} wgrad keys")
        for k, i in keys.items():
            reached.setdefault(k, []).append((plan, i))
            if k not in have:
                missing.setdefault(k, (_id(*plan), i))
    bench = set(BENCHMARKED)
    only_wide = [k for k, by in reached.items() if all(p[0] in WIDE_SIZES for p, _ in by)]
    only_new = [k for k, by in reached.items() if all(p not in bench for p, _ in by)]
    nw_have = sum(1 for k in have if k[0] == "wgrad")
    nw_reached = sum(1 for k in reached if k[0] == "wgrad")
    print(f"{len(reached) - nw_reached} conv and {nw_reached} wgrad keys over the supported plans, {len(have) - nw_have} "
          f"and {nw_have} over the checked launches; {len(only_wide)} reached only by {'/'.join(WIDE_SIZES)}:")
    for k in sorted(only_wide, key=str):
        print(f"  {key_str(k)}   ({', '.join(sorted({_id(*p) for p, _ in reached[k]}))})")
    print(f"{len(only_new)} reached only by the entry-point plans beyond the benchmarked ones:")
    for k in sorted(only_new, key=str):
        print(f"  {key_str(k)}   ({', '.join(sorted({_id(*p) for p, _ in reached[k]}))})")
    for k, (plan, i) in missing.items():
        print(f"MISSING {key_str(k)}: {plan} {i}")
    return missing


def test_every_supported_configuration_is_checked():
    missing = _measured("census", census)
    assert not missing, f"{len(missing)} configurations of supported plans no exact check runs: " + \
        "; ".join(f"{key_str(k)} ({p} {i})" for k, (p, i) in missing.items())
