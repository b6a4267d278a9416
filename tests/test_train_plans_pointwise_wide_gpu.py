"""The BatchNorm, pooling and gradient-routing launches (csrc/bn_train.cu) of the train plans beyond the benchmarked ones,
against fp64, and a census of the launch geometries every supported train plan reaches.

test_train_plans_pointwise_gpu (TP) checks every BatchNorm forward launch and every non-conv backward step of yolov5m b8
1024^2 and yolov5s b2 256x320 (and test_conv_plans_wide_gpu those of yolov5x b8 1024^2).  The plans below reach what those
do not: the P6 graph (four detect_pack / detect_bias levels, SPPF and its max-pool backward on the stride-64 map, 3 x 3 at
192^2 where the 13-wide chained window is wider than the map), odd multi-scale maps carved from a shared arena (P5 17 x 17
at 544^2, P6 9 x 9 at 576^2: pool windows clipped on both sides, pixel counts that leave a partial last reduction block)
and frozen backbones (a pruned backward plan with Concat gradients in channel windows).  Each check is TP's, imported:

  1. every BatchNorm forward launch and every non-conv backward step of each plan, and the accumulate flags of its gradient
     ranges (TP.plan_forward_bn_launches / TP.plan_backward_steps);
  2. the census: a key per pointwise launch, from its arguments alone (nothing runs), restating the launch geometry
     bn_train.cu computes (stat_blocks / colwise_grid with the device's SM count, bnref.stat_layout); every key a supported
     train plan reaches must be reached by a checked plan or by a directed C-ABI case (TP's, and the small cases below for
     keys only unchecked plans reach).

Each case prints its runtime and peak device memory (run with -s)."""
import itertools

import pytest
import torch

from tests import bnref
from tests import test_conv_plans_exact_gpu as CE
from tests import test_conv_plans_wide_gpu as CW
from tests import test_train_plans_pointwise_gpu as TP
from tests.modelgen import build_mirror
from tests.test_p6_gpu import _release_memory
from yolov5_obb_b200.train_backward import BackwardPlan
from yolov5_obb_b200.train_engine import TrainEngine
from yolov5_obb_b200.train_step import freeze_layers

pytestmark = pytest.mark.gpu
DEV = TP.DEV

# ---- 1. the plans: (size, B, H, W, freeze, arena_hw) ------------------------------------------------------------------
WIDE_PLANS = [
    ("x6", 4, 1024, 1024, None, None),        # the widest four-level graph, SPPF on 16 x 16
    ("n6", 1, 192, 192, None, None),          # SPPF and its backward on 3 x 3
    ("s", 2, 544, 544, None, (1024, 1024)),   # multi-scale: odd P5, 17 x 17, in an arena reserved at 1024^2
    ("s6", 2, 576, 576, None, (1024, 1024)),  # multi-scale: odd P6, 9 x 9
    ("s", 2, 256, 256, 10, None),             # --freeze 10: pruned backward
    ("m", 2, 256, 256, 10, None),
]


def _pid(size, B, H, W, freeze=None, arena_hw=None):
    return f"yolov5{size}-b{B}-{H}x{W}" + (f"-freeze{freeze}" if freeze is not None else "") + \
        (f"-arena{arena_hw[0]}x{arena_hw[1]}" if arena_hw is not None else "")


@pytest.mark.parametrize("plan", [pytest.param(p, id=_pid(*p)) for p in WIDE_PLANS])
def test_plan_forward_bn_launches(plan):
    n = CW._measured(f"{_pid(*plan)} BatchNorm forward", TP.plan_forward_bn_launches, *plan)
    print(f"{_pid(*plan)}: {n} BatchNorm launch pairs")


@pytest.mark.parametrize("plan", [pytest.param(p, id=_pid(*p)) for p in WIDE_PLANS])
def test_plan_backward_steps(plan):
    kinds, n_flags = CW._measured(f"{_pid(*plan)} backward steps", TP.plan_backward_steps, *plan)
    print(f"{_pid(*plan)}: step kinds {kinds}; accumulate flags of {n_flags} gradient ranges checked")
    size = plan[0]
    if size.endswith("6"):
        assert kinds["detect_pack"] == 4 and kinds["pool_bwd"] == 1, kinds
    if plan[4] is not None:   # the frozen backbone prunes SPPF's backward and the backbone's BatchNorm backward
        assert "pool_bwd" not in kinds and n_flags > 0, kinds


# ---- 2. the census ------------------------------------------------------------------------------------------------------
STAT_KINDS = ("bn_batch_stats", "bn_sums", "bn_silu_apply", "bn_silu_bwd")
GRID_STRIDE_BLOCKS = 16   # blocks per SM of the grid-stride routing kernels (upsample, max-pool, add, detect pack)


def _loops(total, sms):
    """Whether a grid-stride routing kernel (256 threads, at most 16 blocks per SM) gives a thread several elements."""
    return int(total > 256 * GRID_STRIDE_BLOCKS * sms)


def pointwise_key(kind, a, sms=None):
    """The launch geometry of one pointwise launch, from its arguments only (nothing runs): a tuple (kind, (field,
    value), ...).  a: the launch's arguments by name (npix, C, W, act, ... and the pixel strides / channel offsets of its
    operands).
      BatchNorm kinds (bn_batch_stats and bn_sums: k_bn_stats; bn_silu_apply; bn_silu_bwd: k_bn_bwd_reduce and
      k_bn_bwd_apply): cols (vector columns per pass, hence lanes and idle threads), lanes == 1, more than one column
      group, npix not a multiple of lanes * 16, the reduction saturated at 4 blocks per SM (a thread walks more than 16
      pixels), the element-wise grid saturated at 8 blocks per SM (a thread walks more than one pixel pair), any operand
      with a pixel stride != C, any with a channel offset != 0; apply: SiLU, residual, 2x copy; backward: SiLU, residual
      gradient none / overwrite / accumulate, parameter-gradient accumulate.
      upsample2x_bwd: accumulate.  maxpool5_bwd: map smaller than 5 and than 13 along H and W (the 5-wide window and the
      13-wide chained one clipped on both sides), the gradient form (f32, bf16, both).  add_f32_to_bf16: accumulate,
      strided.  detect_grad_pack: the vector form (no % 4 == 0 and bn % 4 == 0) or the one-channel form, na.
      Every routing kind: whether a thread gets several elements of the grid-stride loop."""
    sms = TP.sms() if sms is None else sms
    if kind in STAT_KINDS:
        npix, C = a["npix"], a["C"]
        vecs, cols, lanes = bnref.stat_layout(C)
        f = [("cols", cols), ("lanes1", int(lanes == 1)), ("groups", int(vecs > cols)),
             ("ragged", int(npix % (lanes * 16) != 0))]
        if kind != "bn_silu_apply":
            f.append(("stat_sat", int(bnref.stat_blocks(npix, C, sms) * lanes * 16 < npix)))
        if kind in ("bn_silu_apply", "bn_silu_bwd"):
            f.append(("col_sat", int(bnref.colwise_grid(npix, C, sms)[0] * 2 * lanes < npix)))
        f += [("strided", int(any(s != C for s in a["strides"]))), ("c_off", int(any(a["coffs"])))]
        if kind == "bn_silu_apply":
            f += [("act", int(a["act"])), ("res", int(a["res"])), ("y2x", int(a["y2x"]))]
        elif kind == "bn_silu_bwd":
            f += [("act", int(a["act"])), ("gres", a["gres"]), ("pacc", int(a["pacc"]))]
    elif kind == "upsample2x_bwd":
        f = [("acc", int(a["acc"])), ("loops", _loops(a["npix"] * (a["C"] // 8), sms))]
    elif kind == "maxpool5_bwd":
        B, H, W, C = a["B"], a["H"], a["W"], a["C"]
        f = [("H<5", int(H < 5)), ("H<13", int(H < 13)), ("W<5", int(W < 5)), ("W<13", int(W < 13)), ("form", a["form"]),
             ("loops", _loops(B * H * W * C, sms))]
    elif kind == "add_f32_to_bf16":
        f = [("acc", int(a["acc"])), ("strided", int(a["stride"] != a["C"])), ("loops", _loops(a["npix"] * a["C"], sms))]
    elif kind == "detect_grad_pack":
        vec4 = a["no"] % 4 == 0 and a["bn"] % 4 == 0
        total = a["B"] * a["H"] * a["W"] * a["na"] * (a["bn"] // 4 if vec4 else a["bn"])
        f = [("vec4", int(vec4)), ("na", a["na"]), ("loops", _loops(total, sms))]
    else:
        raise AssertionError(kind)
    return (kind,) + tuple(f)


def key_str(k):
    return k[0] + " " + " ".join(f"{n}={v}" for n, v in k[1:])


def plan_launches(m, eng, plan):
    """(kind, arguments, what) of every pointwise launch of a train plan: the forward's bn_batch_stats / bn_silu_apply as
    TP._Recorder records them from _forward_eager, then the backward's from the closure defaults of plan.steps."""
    real, rec = eng._L, TP._Recorder()
    eng._L = rec
    try:
        eng._forward_eager(torch.zeros((eng.B, 3) + eng.in_hw, dtype=torch.uint8, device=DEV))
    finally:
        eng._L = real
    stats = [a for n, a in rec.calls if n == "y5obb_bn_batch_stats"]
    apply = [a for n, a in rec.calls if n == "y5obb_bn_silu_apply"]
    assert len(stats) == len(apply) == len(eng.conv_layers)
    out = []
    for i, (lay, sa, aa) in enumerate(zip(eng.conv_layers, stats, apply)):
        z, y = lay.z, lay.y
        assert (sa[0], sa[1], aa[0], aa[10], aa[11]) == (z.ptr, z.pix_stride, z.ptr, y.ptr, y.pix_stride)
        out.append(("bn_batch_stats", dict(npix=sa[2], C=sa[3], strides=(sa[1],), coffs=(z.c_off,)), f"BatchNorm {i}"))
        sl = [z, y] + ([lay.res] if aa[8] is not None else []) + ([lay.y2x] if aa[12] is not None else [])
        out.append(("bn_silu_apply", dict(npix=aa[2], C=aa[3], act=aa[7], res=aa[8] is not None, y2x=aa[12] is not None,
                                          strides=tuple(s.pix_stride for s in sl), coffs=tuple(s.c_off for s in sl)),
                    f"BatchNorm {i}"))
    det = m.model[-1]
    for j, (tag, fn) in enumerate(plan.steps):
        if tag in ("dgrad", "wgrad", "zero"):
            continue
        a, what = TP._defaults(fn), f"backward step {j} ({tag})"
        if tag == "detect_pack":
            out.append(("detect_grad_pack", dict(B=a["dzd"].shape[0], na=det.na, H=a["H"], W=a["W"], no=det.no, bn=a["bn"]),
                        what))
        elif tag == "detect_bias":
            out.append(("bn_sums", dict(npix=a["n"], C=a["C"], strides=(a["C"],), coffs=(0,)), what))
        elif tag == "upsample_bwd":
            out.append(("upsample2x_bwd", dict(npix=a["npix"], C=a["C"], acc=a["acc"]), what))
        elif tag == "pool_bwd":     # three chained 5x5 backward launches (bf16 gradient, then f32 + bf16), then the add
            B = a["npix"] // (a["hh"] * a["ww"])
            for form in ("bf16", "f32+bf16", "f32+bf16"):
                out.append(("maxpool5_bwd", dict(B=B, H=a["hh"], W=a["ww"], C=a["c_"], form=form), what))
            out.append(("add_f32_to_bf16", dict(npix=a["npix"], C=a["c_"], stride=a["ps"], acc=1), what))
        elif tag == "bn_bwd":
            sl = [a["z"], a["gy"]] + ([a["gres"]] if a["gres"] is not None else [])
            gres = "none" if a["gres"] is None else ("acc" if a["gacc"] else "overwrite")
            out.append(("bn_silu_bwd", dict(npix=a["npix"], C=a["C"], act=a["lay"].act, gres=gres, pacc=0,   # (dz: dense)
                                            strides=tuple(s.pix_stride for s in sl) + (a["C"],),
                                            coffs=tuple(s.c_off for s in sl) + (0,)), what))
        else:
            raise AssertionError(f"unexpected backward step {tag}")
    return out


def plan_keys(size, B, H, W, freeze=None, key_only=True):
    """{key: its first launch} of one train plan.  key_only: built on CE.AliasCarver (its buffers alias one allocation):
    keys depend on shapes, strides and channel offsets, never on addresses, and an arena changes only addresses."""
    m = build_mirror(size, nc=15, seed=0).train().to(DEV)
    if freeze is not None:
        freeze_layers(m, [freeze])
    eng = TrainEngine(m, B, H, W, DEV, carver=CE.AliasCarver(torch.device(DEV)) if key_only else None)
    plan = BackwardPlan(eng, TP._trainable(m))
    keys = {}
    for kind, a, what in plan_launches(m, eng, plan):
        keys.setdefault(pointwise_key(kind, a), what)
    del m, eng, plan
    _release_memory()
    return keys


_KEYS = {}   # plan -> plan_keys(plan), built once per module run


def _plan_keys(plan):
    size, B, H, W = plan[:4]
    freeze = plan[4] if len(plan) > 4 else None
    if (size, B, H, W, freeze) not in _KEYS:
        _KEYS[(size, B, H, W, freeze)] = plan_keys(size, B, H, W, freeze)
    return _KEYS[(size, B, H, W, freeze)]


# the train plans the entry points build (test_conv_plans_wide_gpu.SUPPORTED: train.py at 1024^2, its --multi-scale sizes
# and --freeze 10), as (size, B, H, W, freeze)
SUPPORTED = [p[:4] + (p[5] if len(p) > 5 else None,) for p in CW.SUPPORTED if p[4] == "train"]
# the plans whose pointwise launches are checked: TP's, yolov5x (test_conv_plans_wide_gpu) and section 1's
TP_CHECKED = [tuple(p.values) + (None,) for p in TP.PLANS] + [("x", 8, 1024, 1024, None)]
CHECKED = TP_CHECKED + [p[:5] for p in WIDE_PLANS]


def tp_directed():
    """(kind, arguments, case) of TP's C-ABI cases, with the layouts they launch on."""
    out = []
    for C, which, ratio in TP.STAT_CASES + [(48, "8x512x512", r) for r in (0, 10, 100, 300)]:
        npix = 8 * 512 * 512 if which == "8x512x512" else TP.stat_npix(C, which)
        a = dict(npix=npix, C=C, strides=(C + 16,), coffs=(8,))
        out += [("bn_sums", a, f"TP bn_stats C{C} {which}"), ("bn_batch_stats", a, f"TP bn_stats C{C} {which}")]
    for (B, H, W, C), (act, res, up) in itertools.product(TP.APPLY_SHAPES, TP.APPLY_FLAGS):
        st = (C + 16, C + 32) + ((C + 24,) if res else ()) + ((C + 8,) if up else ())
        co = (8, 24) + ((16,) if res else ()) + ((8,) if up else ())
        out.append(("bn_silu_apply", dict(npix=B * H * W, C=C, act=act, res=res, y2x=up, strides=st, coffs=co),
                    f"TP bn_silu_apply {B}x{H}x{W}x{C} act{act} res{res} up{up}"))
    for C, which, ratio, act, gmode, pacc in TP.BWD_CASES:
        npix = 8 * 512 * 512 if which == "8x512x512" else TP.stat_npix(C, which)
        st, co = (C + 16, C + 8, C + 24), (8, 0, 16)
        if gmode is not None:
            st, co = st + (C + 16,), co + (8,)
        gres = "none" if gmode is None else ("acc" if gmode else "overwrite")
        out.append(("bn_silu_bwd", dict(npix=npix, C=C, act=act, gres=gres, pacc=pacc, strides=st, coffs=co),
                    f"TP bn_silu_bwd C{C} {which} gres {gres} pacc {pacc}"))
    for (B, H, W, C), acc in itertools.product(TP.UPSAMPLE_SHAPES, (0, 1)):
        out.append(("upsample2x_bwd", dict(npix=B * H * W, C=C, acc=acc), f"TP upsample2x_bwd {B}x{H}x{W}x{C} acc{acc}"))
    for (npix, C, stride, c_off), acc in itertools.product(TP.ADD_CASES, (0, 1)):
        out.append(("add_f32_to_bf16", dict(npix=npix, C=C, stride=stride, acc=acc), f"TP add_f32_to_bf16 {npix}x{C}"))
    for B, na, H, W, no, bn in TP.PACK_SHAPES:
        out.append(("detect_grad_pack", dict(B=B, na=na, H=H, W=W, no=no, bn=bn), f"TP detect_grad_pack no{no} bn{bn}"))
    for (B, H, W, C), form in itertools.product(TP.POOL_SHAPES, TP.POOL_FORMS):
        out.append(("maxpool5_bwd", dict(B=B, H=H, W=W, C=C, form=form), f"TP maxpool5_bwd {B}x{H}x{W}x{C} {form}"))
    return out


# ---- directed cases: each reaches a key that a supported plan reaches and no checked plan does, at a small shape.  The
# pixel count follows from the case's regime and the device: npix = lanes * 16 * k, plus a tail (1 pixel, 8 for apply) when
# the key is ragged, with k = 2 ("small": neither grid saturated), 2 * SMs ("col": the element-wise grid at its 8 blocks per
# SM, the reduction not) or 4 * SMs + 1 ("stat": both), so a case reaches its key on any SM count.  Layout "dense": every
# operand a whole buffer (pixel stride C, offset 0); "wide": pixel stride C + 16, offset 0; "offset": C + 16, offset 8.
#   ("stats", C, regime, ragged, layout)                          y5obb_bn_stats + y5obb_bn_batch_stats
#   ("apply", C, regime, ragged, act, res, up, layout)            y5obb_bn_silu_apply on a [1, npix / 8, 8, C] map
#   ("bwd", C, regime, ragged, act, gres, layout)                 y5obb_bn_silu_bwd (gres: "none" / "overwrite" / "acc")
# Each was added for a key that only unchecked supported plans reach (yolov5n / l and the P6 models at b8 1024^2, the b16
# multi-scale sizes); the census prints, per key, the case or plan behind it.
DIRECTED = [
    ('stats', 16, 'small', 0, 'dense'), ('stats', 16, 'stat', 0, 'dense'), ('stats', 32, 'stat', 0, 'dense'),
    ('stats', 64, 'stat', 0, 'dense'), ('stats', 64, 'stat', 1, 'dense'), ('stats', 128, 'stat', 0, 'dense'),
    ('stats', 128, 'stat', 1, 'dense'), ('stats', 256, 'stat', 0, 'dense'), ('stats', 256, 'stat', 1, 'dense'),
    ('stats', 288, 'small', 1, 'dense'), ('stats', 384, 'stat', 1, 'dense'), ('stats', 512, 'stat', 0, 'dense'),
    ('stats', 512, 'stat', 1, 'dense'), ('stats', 576, 'small', 1, 'dense'), ('stats', 624, 'stat', 0, 'dense'),
    ('stats', 768, 'small', 1, 'dense'), ('stats', 768, 'stat', 0, 'dense'), ('stats', 768, 'stat', 1, 'dense'),
    ('stats', 1024, 'small', 0, 'dense'), ('apply', 16, 'col', 0, 1, 0, 0, 'dense'),
    ('apply', 16, 'col', 0, 1, 0, 0, 'offset'), ('apply', 16, 'col', 0, 1, 1, 0, 'wide'),
    ('apply', 32, 'col', 0, 1, 0, 0, 'offset'), ('apply', 32, 'col', 0, 1, 1, 0, 'wide'),
    ('apply', 32, 'small', 0, 1, 0, 0, 'wide'), ('apply', 32, 'small', 0, 1, 1, 0, 'dense'),
    ('apply', 64, 'col', 0, 1, 0, 0, 'dense'), ('apply', 64, 'col', 0, 1, 0, 0, 'offset'),
    ('apply', 64, 'col', 0, 1, 0, 0, 'wide'), ('apply', 64, 'col', 0, 1, 1, 0, 'dense'),
    ('apply', 64, 'col', 0, 1, 1, 0, 'wide'), ('apply', 64, 'col', 1, 1, 0, 0, 'dense'),
    ('apply', 64, 'col', 1, 1, 0, 0, 'offset'), ('apply', 64, 'col', 1, 1, 0, 0, 'wide'),
    ('apply', 64, 'col', 1, 1, 1, 0, 'dense'), ('apply', 64, 'col', 1, 1, 1, 0, 'wide'),
    ('apply', 64, 'small', 0, 1, 0, 1, 'offset'), ('apply', 128, 'col', 0, 1, 0, 0, 'dense'),
    ('apply', 128, 'col', 0, 1, 0, 0, 'offset'), ('apply', 128, 'col', 0, 1, 0, 0, 'wide'),
    ('apply', 128, 'col', 0, 1, 0, 1, 'offset'), ('apply', 128, 'col', 0, 1, 1, 0, 'dense'),
    ('apply', 128, 'col', 0, 1, 1, 0, 'wide'), ('apply', 128, 'col', 1, 1, 0, 0, 'dense'),
    ('apply', 128, 'col', 1, 1, 0, 0, 'offset'), ('apply', 128, 'col', 1, 1, 0, 0, 'wide'),
    ('apply', 128, 'col', 1, 1, 0, 1, 'offset'), ('apply', 128, 'col', 1, 1, 1, 0, 'dense'),
    ('apply', 128, 'col', 1, 1, 1, 0, 'wide'), ('apply', 256, 'col', 0, 1, 0, 0, 'dense'),
    ('apply', 256, 'col', 0, 1, 0, 0, 'offset'), ('apply', 256, 'col', 0, 1, 0, 0, 'wide'),
    ('apply', 256, 'col', 0, 1, 0, 1, 'offset'), ('apply', 256, 'col', 0, 1, 1, 0, 'dense'),
    ('apply', 256, 'col', 0, 1, 1, 0, 'wide'), ('apply', 256, 'col', 1, 1, 0, 0, 'dense'),
    ('apply', 256, 'col', 1, 1, 0, 0, 'offset'), ('apply', 256, 'col', 1, 1, 0, 0, 'wide'),
    ('apply', 256, 'col', 1, 1, 0, 1, 'offset'), ('apply', 256, 'col', 1, 1, 1, 0, 'wide'),
    ('apply', 288, 'small', 1, 1, 0, 0, 'dense'), ('apply', 288, 'small', 1, 1, 0, 0, 'offset'),
    ('apply', 288, 'small', 1, 1, 0, 0, 'wide'), ('apply', 288, 'small', 1, 1, 1, 0, 'dense'),
    ('apply', 288, 'small', 1, 1, 1, 0, 'wide'), ('apply', 384, 'col', 1, 1, 0, 0, 'wide'),
    ('apply', 384, 'col', 1, 1, 0, 1, 'offset'), ('apply', 384, 'col', 1, 1, 1, 0, 'dense'),
    ('apply', 384, 'col', 1, 1, 1, 0, 'wide'), ('apply', 512, 'col', 0, 1, 0, 0, 'dense'),
    ('apply', 512, 'col', 0, 1, 0, 0, 'offset'), ('apply', 512, 'col', 1, 1, 0, 0, 'dense'),
    ('apply', 512, 'small', 0, 1, 0, 0, 'offset'), ('apply', 512, 'small', 0, 1, 0, 0, 'wide'),
    ('apply', 512, 'small', 0, 1, 0, 1, 'offset'), ('apply', 512, 'small', 0, 1, 1, 0, 'dense'),
    ('apply', 512, 'small', 0, 1, 1, 0, 'wide'), ('apply', 576, 'col', 1, 1, 0, 0, 'dense'),
    ('apply', 576, 'col', 1, 1, 0, 0, 'offset'), ('apply', 576, 'small', 1, 1, 0, 0, 'wide'),
    ('apply', 576, 'small', 1, 1, 0, 1, 'offset'), ('apply', 768, 'col', 0, 1, 0, 0, 'offset'),
    ('apply', 768, 'col', 1, 1, 0, 0, 'dense'), ('apply', 768, 'small', 0, 1, 0, 0, 'wide'),
    ('apply', 768, 'small', 0, 1, 0, 1, 'offset'), ('apply', 960, 'col', 0, 1, 0, 0, 'dense'),
    ('apply', 960, 'col', 0, 1, 0, 0, 'offset'), ('apply', 1024, 'col', 0, 1, 0, 0, 'dense'),
    ('apply', 1024, 'small', 0, 1, 0, 0, 'dense'), ('bwd', 16, 'col', 0, 1, 'none', 'dense'),
    ('bwd', 16, 'col', 0, 1, 'none', 'offset'), ('bwd', 16, 'col', 0, 1, 'overwrite', 'wide'),
    ('bwd', 16, 'stat', 0, 1, 'none', 'dense'), ('bwd', 32, 'col', 0, 1, 'none', 'offset'),
    ('bwd', 32, 'col', 0, 1, 'overwrite', 'wide'), ('bwd', 32, 'small', 0, 1, 'none', 'wide'),
    ('bwd', 32, 'small', 0, 1, 'overwrite', 'dense'), ('bwd', 32, 'stat', 0, 1, 'none', 'dense'),
    ('bwd', 32, 'stat', 0, 1, 'none', 'offset'), ('bwd', 32, 'stat', 0, 1, 'overwrite', 'wide'),
    ('bwd', 48, 'col', 1, 1, 'none', 'dense'), ('bwd', 48, 'col', 1, 1, 'none', 'offset'),
    ('bwd', 48, 'col', 1, 1, 'overwrite', 'dense'), ('bwd', 48, 'col', 1, 1, 'overwrite', 'wide'),
    ('bwd', 64, 'col', 0, 1, 'none', 'dense'), ('bwd', 64, 'col', 0, 1, 'none', 'offset'),
    ('bwd', 64, 'col', 0, 1, 'none', 'wide'), ('bwd', 64, 'col', 0, 1, 'overwrite', 'dense'),
    ('bwd', 64, 'col', 0, 1, 'overwrite', 'wide'), ('bwd', 64, 'col', 1, 1, 'none', 'dense'),
    ('bwd', 64, 'col', 1, 1, 'none', 'offset'), ('bwd', 64, 'col', 1, 1, 'none', 'wide'),
    ('bwd', 64, 'col', 1, 1, 'overwrite', 'dense'), ('bwd', 64, 'col', 1, 1, 'overwrite', 'wide'),
    ('bwd', 64, 'stat', 0, 1, 'none', 'dense'), ('bwd', 64, 'stat', 0, 1, 'none', 'offset'),
    ('bwd', 64, 'stat', 0, 1, 'none', 'wide'), ('bwd', 64, 'stat', 0, 1, 'overwrite', 'dense'),
    ('bwd', 64, 'stat', 0, 1, 'overwrite', 'wide'), ('bwd', 64, 'stat', 1, 1, 'none', 'dense'),
    ('bwd', 64, 'stat', 1, 1, 'none', 'offset'), ('bwd', 64, 'stat', 1, 1, 'none', 'wide'),
    ('bwd', 64, 'stat', 1, 1, 'overwrite', 'dense'), ('bwd', 64, 'stat', 1, 1, 'overwrite', 'wide'),
    ('bwd', 96, 'stat', 1, 1, 'none', 'offset'), ('bwd', 96, 'stat', 1, 1, 'none', 'wide'),
    ('bwd', 96, 'stat', 1, 1, 'overwrite', 'dense'), ('bwd', 96, 'stat', 1, 1, 'overwrite', 'wide'),
    ('bwd', 128, 'col', 0, 1, 'none', 'dense'), ('bwd', 128, 'col', 0, 1, 'none', 'offset'),
    ('bwd', 128, 'col', 0, 1, 'none', 'wide'), ('bwd', 128, 'col', 0, 1, 'overwrite', 'dense'),
    ('bwd', 128, 'col', 0, 1, 'overwrite', 'wide'), ('bwd', 128, 'small', 0, 1, 'overwrite', 'dense'),
    ('bwd', 128, 'small', 0, 1, 'overwrite', 'wide'), ('bwd', 128, 'stat', 0, 1, 'none', 'dense'),
    ('bwd', 128, 'stat', 0, 1, 'none', 'offset'), ('bwd', 128, 'stat', 0, 1, 'none', 'wide'),
    ('bwd', 128, 'stat', 0, 1, 'overwrite', 'dense'), ('bwd', 128, 'stat', 0, 1, 'overwrite', 'wide'),
    ('bwd', 128, 'stat', 1, 1, 'none', 'dense'), ('bwd', 128, 'stat', 1, 1, 'none', 'offset'),
    ('bwd', 128, 'stat', 1, 1, 'none', 'wide'), ('bwd', 128, 'stat', 1, 1, 'overwrite', 'dense'),
    ('bwd', 128, 'stat', 1, 1, 'overwrite', 'wide'), ('bwd', 192, 'small', 1, 1, 'overwrite', 'dense'),
    ('bwd', 192, 'stat', 1, 1, 'none', 'wide'), ('bwd', 192, 'stat', 1, 1, 'overwrite', 'dense'),
    ('bwd', 192, 'stat', 1, 1, 'overwrite', 'wide'), ('bwd', 256, 'col', 0, 1, 'none', 'dense'),
    ('bwd', 256, 'col', 0, 1, 'none', 'offset'), ('bwd', 256, 'col', 0, 1, 'none', 'wide'),
    ('bwd', 256, 'col', 0, 1, 'overwrite', 'dense'), ('bwd', 256, 'col', 0, 1, 'overwrite', 'wide'),
    ('bwd', 256, 'col', 1, 1, 'none', 'dense'), ('bwd', 256, 'col', 1, 1, 'none', 'offset'),
    ('bwd', 256, 'col', 1, 1, 'none', 'wide'), ('bwd', 256, 'col', 1, 1, 'overwrite', 'wide'),
    ('bwd', 256, 'small', 0, 1, 'overwrite', 'wide'), ('bwd', 256, 'stat', 0, 1, 'none', 'dense'),
    ('bwd', 256, 'stat', 0, 1, 'none', 'offset'), ('bwd', 256, 'stat', 1, 1, 'none', 'dense'),
    ('bwd', 256, 'stat', 1, 1, 'none', 'offset'), ('bwd', 288, 'small', 1, 1, 'none', 'dense'),
    ('bwd', 288, 'small', 1, 1, 'none', 'offset'), ('bwd', 288, 'small', 1, 1, 'none', 'wide'),
    ('bwd', 288, 'small', 1, 1, 'overwrite', 'dense'), ('bwd', 288, 'small', 1, 1, 'overwrite', 'wide'),
    ('bwd', 384, 'col', 1, 1, 'none', 'wide'), ('bwd', 384, 'col', 1, 1, 'overwrite', 'dense'),
    ('bwd', 384, 'col', 1, 1, 'overwrite', 'wide'), ('bwd', 384, 'stat', 1, 1, 'none', 'dense'),
    ('bwd', 384, 'stat', 1, 1, 'none', 'offset'), ('bwd', 512, 'col', 0, 1, 'none', 'dense'),
    ('bwd', 512, 'col', 0, 1, 'none', 'offset'), ('bwd', 512, 'small', 0, 1, 'none', 'offset'),
    ('bwd', 512, 'small', 0, 1, 'none', 'wide'), ('bwd', 512, 'small', 0, 1, 'overwrite', 'dense'),
    ('bwd', 512, 'small', 0, 1, 'overwrite', 'wide'), ('bwd', 512, 'stat', 0, 1, 'none', 'dense'),
    ('bwd', 512, 'stat', 1, 1, 'none', 'dense'), ('bwd', 576, 'col', 1, 1, 'none', 'dense'),
    ('bwd', 576, 'col', 1, 1, 'none', 'offset'), ('bwd', 576, 'small', 1, 1, 'none', 'offset'),
    ('bwd', 576, 'small', 1, 1, 'none', 'wide'), ('bwd', 768, 'col', 0, 1, 'none', 'offset'),
    ('bwd', 768, 'col', 1, 1, 'none', 'dense'), ('bwd', 768, 'small', 0, 1, 'none', 'offset'),
    ('bwd', 768, 'small', 0, 1, 'none', 'wide'), ('bwd', 768, 'stat', 0, 1, 'none', 'dense'),
    ('bwd', 768, 'stat', 1, 1, 'none', 'dense'), ('bwd', 960, 'col', 0, 1, 'none', 'dense'),
    ('bwd', 960, 'col', 0, 1, 'none', 'offset'), ('bwd', 1024, 'col', 0, 1, 'none', 'dense'),
    ('bwd', 1024, 'small', 0, 1, 'none', 'dense'),
]

_LAYOUT = {"dense": (0, 0), "wide": (16, 0), "offset": (16, 8)}


def directed_npix(case, sms=None):
    sms = TP.sms() if sms is None else sms
    C, regime, ragged = case[1:4]
    k = {"small": 2, "col": 2 * sms, "stat": 4 * sms + 1}[regime]
    return bnref.stat_layout(C)[2] * 16 * k + ((8 if case[0] == "apply" else 1) if ragged else 0)


def directed_launches(case, sms=None):
    """(kind, arguments) of one directed case, as pointwise_key reads them."""
    C, npix = case[1], directed_npix(case, sms)
    extra, c_off = _LAYOUT[case[-1]]
    if case[0] == "stats":
        a = dict(npix=npix, C=C, strides=(C + extra,), coffs=(c_off,))
        return [("bn_sums", a), ("bn_batch_stats", a)]
    if case[0] == "apply":
        act, res, up = case[4:7]
        n = 2 + bool(res) + bool(up)
        return [("bn_silu_apply", dict(npix=npix, C=C, act=act, res=res, y2x=up, strides=(C + extra,) * n,
                                       coffs=(c_off,) * n))]
    if case[0] == "bwd":
        act, gres = case[4:6]
        n = 3 + (gres != "none")
        return [("bn_silu_bwd", dict(npix=npix, C=C, act=act, gres=gres, pacc=0, strides=(C + extra,) * n,
                                     coffs=(c_off,) * n))]
    raise AssertionError(case)


def _directed_id(case):
    return "-".join(map(str, case))


@pytest.mark.parametrize("case", [pytest.param(c, id=_directed_id(c)) for c in DIRECTED])
def test_directed_case(case):
    """The launch with TP's data and TP's checks, on the case's layout."""
    extra, c_off = _LAYOUT[case[-1]]
    C, npix = case[1], directed_npix(case)
    if case[0] == "stats":
        g = torch.Generator(device=DEV).manual_seed(C * 7 + npix)
        zbuf, zv = TP.slab((npix,), C, extra=extra, c_off=c_off, fill=TP.IN_SENT)
        zv.copy_(TP.gen_z((npix,), C, 10, g))
        bn = TP.rand_bn(C, g)
        s, q, out = TP.run_stats(zv, zbuf.shape[-1], npix, C, bn)
        TP.check_sums(zv, npix, C, s, q, "directed bn_stats sums")
        TP.check_batch_stats(zv, npix, C, s, q, bn, out, 10, "directed bn_batch_stats")
    elif case[0] == "apply":
        act, res, up = case[4:7]
        B, H, W = 1, npix // 8, 8
        g = torch.Generator(device=DEV).manual_seed(npix + C)
        zbuf, zv = TP.slab((B, H, W), C, extra=extra, c_off=c_off, fill=TP.IN_SENT)
        zv.copy_(TP.gen_z((B, H, W), C, 2.0, g))
        _, _, st = TP.run_stats(zv, zbuf.shape[-1], npix, C, TP.rand_bn(C, g))
        rbuf = rv = None
        if res:
            rbuf, rv = TP.slab((B, H, W), C, extra=extra, c_off=c_off, fill=TP.IN_SENT)
            rv.copy_(torch.randn(B, H, W, C, device=DEV, generator=g).bfloat16())
        ybuf, yv = TP.slab((B, H, W), C, extra=extra, c_off=c_off)
        y_before = ybuf.clone()
        ubuf = uv = u_before = None
        if up:
            ubuf, uv = TP.slab((B, 2 * H, 2 * W), C, extra=extra, c_off=c_off)
            u_before = ubuf.clone()
        assert TP.lib().y5obb_bn_silu_apply(zv.data_ptr(), zbuf.shape[-1], npix, C, W, st["scale"].data_ptr(),
                                            st["shift"].data_ptr(), act, rv.data_ptr() if res else None,
                                            rbuf.shape[-1] if res else 0, yv.data_ptr(), ybuf.shape[-1],
                                            uv.data_ptr() if up else None, ubuf.shape[-1] if up else 0, TP.stream()) == 0
        torch.cuda.synchronize()
        TP.check_apply(zv, st["scale"], st["shift"], act, rv, yv, ybuf, y_before, c_off,
                       (ubuf, u_before, c_off) if up else None, "directed bn_silu_apply")
    elif case[0] == "bwd":
        act, gres = case[4:6]
        g = torch.Generator(device=DEV).manual_seed(C + npix)
        zbuf, zv = TP.slab((npix,), C, extra=extra, c_off=c_off, fill=TP.IN_SENT)
        zv.copy_(TP.gen_z((npix,), C, 3, g))
        _, _, st = TP.run_stats(zv, zbuf.shape[-1], npix, C, TP.rand_bn(C, g))
        dbuf, dyv = TP.slab((npix,), C, extra=extra, c_off=c_off, fill=TP.IN_SENT)
        dyv.copy_(torch.randn(npix, C, device=DEV, generator=g).bfloat16())
        dzbuf, dzv = TP.slab((npix,), C, extra=extra, c_off=c_off)
        dz_before = dzbuf.clone()
        gbuf = gv = g_before = None
        if gres != "none":
            gbuf, gv = TP.slab((npix,), C, extra=extra, c_off=c_off)
            if gres == "acc":
                gv.copy_(torch.randn(npix, C, device=DEV, generator=g).bfloat16())
            g_before = gbuf.clone()
        s1, s2 = TP.f32(C), TP.f32(C)
        dg, db = torch.randn(C, device=DEV, generator=g), torch.randn(C, device=DEV, generator=g)
        odg, odb = dg.clone(), db.clone()
        scr = TP.scratch(C)
        assert TP.lib().y5obb_bn_silu_bwd(zv.data_ptr(), zbuf.shape[-1], dyv.data_ptr(), dbuf.shape[-1], npix, C,
                                          st["scale"].data_ptr(), st["shift"].data_ptr(), st["mean"].data_ptr(),
                                          st["invstd"].data_ptr(), act, s1.data_ptr(), s2.data_ptr(), dzv.data_ptr(),
                                          dzbuf.shape[-1], gv.data_ptr() if gv is not None else None,
                                          gbuf.shape[-1] if gbuf is not None else 0, int(gres == "acc"), dg.data_ptr(),
                                          db.data_ptr(), 0, scr.data_ptr(), scr.numel(), TP.stream()) == 0
        torch.cuda.synchronize()
        TP.unchanged(dzbuf, dz_before, TP.chan_mask(dzbuf, c_off, C), "directed bn_silu_bwd dz")
        gr = None
        if gbuf is not None:
            TP.unchanged(gbuf, g_before, TP.chan_mask(gbuf, c_off, C), "directed bn_silu_bwd gres")
            gr = (gv, g_before[..., c_off:c_off + C], gres == "acc")
        TP.check_bwd(zv, dyv, st, act, s1, s2, dzv, gr, (dg, db, odg, odb, 0), "directed bn_silu_bwd")
    else:
        raise AssertionError(case)


def census(checked=CHECKED, supported=SUPPORTED, directed=True, extra=DIRECTED):
    """-> (missing, reached): missing {key: (plan, launch)} of every key the supported plans reach that no checked plan,
    no TP C-ABI case (directed=True) and no case of `extra` reaches; reached {key: [supported plans]}.  Prints each key the
    supported plans reach with the checked plan or directed case behind it, and the keys only section 1's plans check."""
    have = {}
    for plan in checked:
        for k in _plan_keys(plan):
            have.setdefault(k, []).append(_pid(*plan))
    if directed:
        for kind, a, what in tp_directed():
            have.setdefault(pointwise_key(kind, a), []).append(what)
    for case in extra:
        for kind, a in directed_launches(case):
            have.setdefault(pointwise_key(kind, a), []).append(f"directed {_directed_id(case)}")
    reached, missing = {}, {}
    print("\npointwise keys per supported train plan:")
    for plan in supported:
        keys = _plan_keys(plan)
        print(f"  {_pid(*plan):40s} {len(keys):3d} keys")
        for k, i in keys.items():
            reached.setdefault(k, []).append(_pid(*plan))
            if k not in have:
                missing.setdefault(k, (_pid(*plan), i))
    print(f"{len(reached)} keys over the supported plans, {len(have)} over the checked launches; behind each key:")
    for k in sorted(reached, key=str):
        print(f"  {key_str(k)}: {have[k][0] if k in have else 'NOTHING'}")
    wide = {_pid(*p[:5]) for p in WIDE_PLANS}
    only = [k for k in reached if k in have and set(have[k]) <= wide]
    print(f"{len(only)} keys of supported plans checked only by section 1's plans:")
    for k in sorted(only, key=str):
        print(f"  {key_str(k)}   (checked by {', '.join(have[k])}; reached by {', '.join(reached[k])})")
    for k, (plan, i) in missing.items():
        print(f"MISSING {key_str(k)}: {plan} {i}")
    return missing, reached


def test_alias_built_plans_key_like_allocated_ones():
    """The census reads train plans built on aliased buffers: their pointwise launches key exactly as those of the same plan
    on its own buffers."""
    for plan in [("n", 2, 96, 160, None), ("s", 2, 128, 128, 10)]:
        assert plan_keys(*plan, key_only=False) == plan_keys(*plan, key_only=True), plan


def test_every_supported_pointwise_configuration_is_checked():
    missing, reached = CW._measured("pointwise census", census)
    assert not missing, f"{len(missing)} pointwise launch geometries of supported plans no check runs: " + \
        "; ".join(f"{key_str(k)} ({p} {i})" for k, (p, i) in missing.items())


def test_census_fails_without_the_wide_plans():
    """The census has teeth: without section 1's plans and the directed cases it fails, and among what it names is a key
    only P6 plans reach."""
    missing, reached = CW._measured("pointwise census without section 1 and the directed cases", census, TP_CHECKED,
                                    SUPPORTED, False, [])
    assert missing
    p6 = [k for k in missing if all(p.split("-")[0].endswith("6") for p in reached[k])]
    assert p6, "no missing key is reached by P6 plans only"
    print(f"{len(missing)} keys missing, {len(p6)} of them reached only by P6 plans, e.g. {key_str(p6[0])}")
