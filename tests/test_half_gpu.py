"""fp16 inference plans (a model whose parameters are fp16, `model.half()`) on the GPU.

  * every conv launch of the fp16 plans in CHECKED_F16 (every size's eval and records plans, test-time augmentation, scene
    tiles, a letterboxed shape), on integer operands: conv outputs equal their descriptor's fp64 value rounded once to
    fp16 (tests/convref.py, SiLU layers within its bound with the fp16 rounding in place of the bf16 one), Detect launches equal models/yolo.py:63-77 restated in
    torch on a half tensor, applied to a raw-logit launch of the same conv, bit for bit;
  * the same decode on the plan's own logits of a calibrated model, with theta logits that tie after the sigmoid's rounding;
  * records through non_max_suppression_obb against the oracle NMS fed the reference's half arithmetic;
  * the stem input (uint8 and fp32 images) and the test-time-augmentation resample against torch half compositions;
  * the distance of the plan's rows from the fp32 eager forward, against the bf16 plan's and torch's own half forward's;
  * the letterbox and scene-tile staging against torch half compositions, the pipeline and whole scenes on a half model;
  * the validation loss of an fp16 plan against ComputeLoss on the fp16-rounded logits, bit for bit, and the Validator;
  * a census: every kernel configuration the supported fp16 plans reach is reached by an exactly checked plan.
"""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.eager_ref import EagerFusedModel
from oracle.postprocess import non_max_suppression_obb as oracle_nms
from tests.modelgen import build_mirror, calibrated_bench_model
from oracle import loss_ref
from tests import convref
from tests.convref import conv_reference
from tests.test_conv_plans_exact_gpu import IN_SENT, LIMIT, OUT_SENT, _compare, _real_rows, bits, rint
from tests.tilegen import synth_tiles
from yolov5_obb_b200.conv import F16, MODE_DETECT, Conv as ConvOp, WindowView
from yolov5_obb_b200.engine import TTA_SCALES, InferenceEngine, TTAPlan
from yolov5_obb_b200.general import DetectRecords, half_threshold, non_max_suppression_obb

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FP16_REL = 2.0 ** -11    # one fp16 rounding to nearest: half an ulp is at most 2^-11 of the value

# torch's half forward (oracle/eager_ref.py, cuDNN) is this many times closer to the fp32 forward than the fp16 plan may be
# at most; measured on an H100 80GB HBM3 (700 W): see test_plan_distance_from_fp32
HALF_EAGER_MULTIPLE = 1.5   # measured: 0.99 (fp16 plan 3.72e-3, torch half 3.77e-3, bf16 plan 2.56e-2)


@pytest.fixture(scope="module")
def calibrated():
    """A calibrated yolov5s (CPU, fp32); tests take copies."""
    return calibrated_bench_model("s", nc=15)


def half_mirror(size, seed=0, **kw):
    return build_mirror(size, nc=15, seed=seed, **kw).half().to(DEV)


def raw_twin(op, raw):
    """A raw-logit launch (det_decode 0) of a Detect op: same input slice, weights, bias and rows, into `raw` (fp16)."""
    x, wp, bp, out, res, out2x, det = op._keep
    d = dict(det, out=raw, decode=False, descale=None)
    return ConvOp(x, wp, bp, op.desc.Cout, 1, 1, 0, False, det=d, flags=F16, bias_prehalved=True)


def decode_rows(raw, det, descale=None):
    """models/yolo.py:63-77 on the half tensor of one Detect op's raw logits (its [B, rows, no] row range), and
    _descale_pred (models/yolo.py:183-198) for a test-time-augmentation branch."""
    d = det
    B, no = raw.shape[0], d["no"]
    na = len(d["anchors_px"]) // 2
    n = raw.shape[1]
    hw = n // na
    H, W = d["_hw"]
    assert H * W == hw
    x = raw.view(B, na, H, W, no)
    yv, xv = torch.meshgrid(torch.arange(H, device=DEV), torch.arange(W, device=DEV), indexing="ij")
    grid = torch.stack((xv, yv), 2).expand((1, na, H, W, 2)).float()
    ag = torch.tensor(d["anchors_px"], dtype=torch.float32, device=DEV).view(1, na, 1, 1, 2).expand((1, na, H, W, 2))
    stride = torch.tensor(d["stride"], dtype=torch.float32, device=DEV)
    y = x.sigmoid()
    y[..., 0:2] = (y[..., 0:2] * 2 - 0.5 + grid) * stride
    y[..., 2:4] = (y[..., 2:4] * 2) ** 2 * ag
    y = y.view(B, -1, no)
    if descale is not None:   # (the plan's fp32 1 / s: the branch's scale s is the TTA_SCALES entry it came from)
        inv, flip_w = descale
        s = next(s for s in TTA_SCALES if float(np.float32(1) / np.float32(s)) == inv)
        y[..., :4] /= s
        if flip_w > 0:
            y[..., 0] = flip_w - y[..., 0]
    return y


def detect_view(op):
    d = op.desc
    det = op._keep[6]
    no = d.det_no
    rw = ((no - 180 + 1) + 3) // 4 * 4 if d.det_decode == 2 else no
    buf = det["out"]
    na = d.Cout // no
    rows = na * d.Hin * d.Win
    return buf[:, d.det_row_off:d.det_row_off + rows], dict(det, _hw=(d.Hin, d.Win))


def check_detect(op, raw_buf, st, what, integer=True):
    """Runs the raw twin and the op; the op's rows (or records) must equal the torch half decode of the twin's logits."""
    d = op.desc
    view, det = detect_view(op)
    twin = raw_twin(op, raw_buf)
    if integer:
        x, wp, bp = op._keep[:3]
        x.view().copy_(rint(x.view().shape, 2))
        na, no = d.Cout // d.det_no, d.det_no
        bn = wp.shape[1] // na
        rows = torch.tensor([a * bn + j for a in range(na) for j in range(no)], device=DEV)
        wv = rint((wp.shape[0], len(rows), d.Cin), 1) * (torch.rand((wp.shape[0], len(rows), d.Cin), device=DEV) < 4.0 / d.Cin)
        wp[:, rows, :d.Cin] = wv.half()
        bp.zero_()
        bp[rows] = rint((len(rows),), 2)
        raw_buf.fill_(OUT_SENT)
        # the exact logits of the 1x1 conv, in the output's row order (a, h, w)
        xin = x.view().double()
        lg = xin @ wp[0, rows, :d.Cin].double().t() + bp[rows].double()
        exact = lg.view(d.B, d.Hin, d.Win, na, no).permute(0, 3, 1, 2, 4).reshape(d.B, -1, no)
    twin.run()
    view.fill_(OUT_SENT)
    op.run()
    torch.cuda.synchronize()
    raw_rows = raw_buf[:, d.det_row_off:d.det_row_off + view.shape[1]]
    if integer:   # the raw launch: the exact logits rounded once to fp16
        assert torch.equal(bits(raw_rows), bits(exact.float().half())), f"{what}: raw logits"
    rows16 = decode_rows(raw_rows.clone(), det, det.get("descale"))
    nfix = d.det_no - 180
    if d.det_decode == 2:
        rec = view
        assert torch.equal(bits(rec[..., :nfix]), bits(rows16[..., :nfix].float())), f"{what}: record columns"
        th = torch.max(rows16[..., nfix:], -1).indices.float()
        assert torch.equal(rec[..., nfix], th), f"{what}: theta index"
        assert not rec[..., nfix + 1:].any(), f"{what}: record padding"
        lg = raw_rows[..., nfix:].float()
        st["theta_moved"] += int((lg.argmax(-1).float() != th).sum())
    else:
        assert torch.equal(bits(view), bits(rows16)), f"{what}: eval rows, " \
            f"{int((bits(view) != bits(rows16)).sum())} differ"
    st["detect"] += 1


def check_conv16(op, st, what):
    """tests/test_conv_plans_exact_gpu.check_conv for an fp16 launch: integer operands (exact in fp16), sentinels around
    the read and written regions, tests/convref.py's fp64 evaluation of the descriptor, one rounding to fp16."""
    d = op.desc
    x, wp, bp, out, res, out2x, det = op._keep
    dests = ([out.buf] if out is not None else []) + ([out2x.buf] if out2x is not None else [])
    for t in dests:
        t.fill_(OUT_SENT)
    rx, rw, rb = (2, 1, 4) if d.act else (8, 8, 8)
    if isinstance(x, WindowView):   # the stem's window view
        x.buf.copy_(rint(x.buf.shape, rx))
    else:
        if all(x.buf.data_ptr() != t.data_ptr() for t in dests):
            x.buf.fill_(IN_SENT)
        x.view().copy_(rint(x.view().shape, rx))
    rows = _real_rows(d, wp)
    wv = rint((wp.shape[0], len(rows), d.Cin), rw)
    wp[:, rows, :d.Cin] = wv.half()
    b = rint((len(rows),), rb)
    bp.zero_()
    bp[rows] = b * 0.5 if d.act else b    # the buffer holds 0.5 * bias (Y5OBB_CONV_BIAS_HALVED)
    rr = 0
    if res is not None:
        rr = 8
        res.view().copy_(rint(res.view().shape, rr))
    assert wp.shape[0] * d.Cin * rx * (wv.abs().max().item()) + rb + rr < LIMIT
    # convref's SiLU bound ends with one bf16 rounding of the stored value (2^-8); an fp16 store rounds to 2^-11
    saved, convref.BF16_REL = convref.BF16_REL, FP16_REL
    try:
        recs = conv_reference(op)
    finally:
        convref.BF16_REL = saved
    before = {t.data_ptr(): t.clone() for t in (r.buf for r in recs)}
    op.run()
    torch.cuda.synchronize()
    exact, worst = _compare(recs, before, what)
    st["conv"] += 1
    st["bitwise" if exact else "tolerance"] += 1
    st["worst"] = max(st["worst"], worst)


def check_plan(eng, what, st):
    raw = torch.empty(eng.pred.shape[:2] + (eng.no,), dtype=torch.float16, device=DEV)
    for k, op in enumerate(eng.convs):
        if op.desc.mode == MODE_DETECT:
            check_detect(op, raw, st, f"{what} op {k}")
        else:
            assert op.desc.flags & F16
            check_conv16(op, st, f"{what} op {k}")


def _stats():
    return dict(conv=0, bitwise=0, tolerance=0, worst=0.0, ties=0, rows=0, detect=0, theta_moved=0)


_MODELS = {}


def half_model(size):
    if size not in _MODELS:
        _MODELS[size] = half_mirror(size)
    return _MODELS[size]


def build_plan(size, B, H, W, kind):
    """The engines of one fp16 plan as the half entry points build it: Model.forward ("forward"), detect_records / records_plan
    ("records"), forward_augment ("tta") and detect_records(augment=True) ("tta-records")."""
    m = half_model(size)
    if kind in ("forward", "records"):
        return [InferenceEngine(m, B, H, W, DEV, compact_detect=kind == "records")]
    return TTAPlan(m, B, H, W, DEV, compact_detect=kind == "tta-records").engines


def _pid(plan):
    return "{}-b{}-{}x{}-{}".format(*plan)


# The fp16 plans every launch of which is checked exactly (test_every_fp16_launch_matches_its_descriptor)
CHECKED_F16 = [(s, 16, 1024, 1024, k) for s in "nsmlx" for k in ("forward", "records")] + \
              [(s + "6", 8, 1280, 1280, k) for s in "nsmlx" for k in ("forward", "records")] + \
              [("s", 16, 1024, 1024, k) for k in ("tta", "tta-records")] + \
              [("n6", 16, 1280, 1280, "forward"), ("x6", 16, 1280, 1280, "forward")] + \
              [("s", 16, 1056, 1056, "records"), ("s6", 16, 1088, 1088, "records"), ("s", 1, 1024, 576, "records"),
               ("s", 1, 320, 1024, "records")]
# The fp16 plans the half entry points build (test_every_fp16_configuration_is_checked keys them without running them):
# forward and records of every size at its benchmark batch, SceneDetector tiles (1056^2, 1088^2 with a P6 model),
# run_images' letterboxed shapes, test-time augmentation.  An ensemble's members are these plans at the same shapes.
SUPPORTED_F16 = [(s, 16, 1024, 1024, k) for s in "nsmlx" for k in ("forward", "records")] + \
                [(s + "6", 16, 1280, 1280, k) for s in "nsmlx" for k in ("forward", "records")] + \
                [(s, 16, 1024, 1024, k) for s in "sm" for k in ("tta", "tta-records")] + \
                [("s", 16, 1056, 1056, "records"), ("x", 16, 1056, 1056, "records"), ("s6", 16, 1088, 1088, "records"),
                 ("s", 1, 1024, 576, "records"), ("s", 1, 320, 1024, "records")]


@pytest.mark.parametrize("plan", CHECKED_F16, ids=_pid)
def test_every_fp16_launch_matches_its_descriptor(plan):
    st = _stats()
    engines = build_plan(*plan)
    for k, eng in enumerate(engines):
        check_plan(eng, f"{_pid(plan)} engine {k}", st)
    del engines
    torch.cuda.empty_cache()
    print(f"{_pid(plan)}: {st}")
    assert st["conv"] > 20 and st["detect"] >= 2


def f16_key(op):
    """conv_key (tests/test_conv_plans_wide_gpu.py) of an fp16 launch, with the element type in the key."""
    from tests.test_conv_plans_wide_gpu import conv_key
    assert op.desc.flags & F16
    return ("f16",) + conv_key(op)


def _plan_keys(plan):
    engines = build_plan(*plan)
    keys = {}
    for k, eng in enumerate(engines):
        for i, op in enumerate(eng.convs):
            keys.setdefault(f16_key(op), f"{_pid(plan)} engine {k} launch {i}")
    del engines
    torch.cuda.empty_cache()
    return keys


def test_every_fp16_configuration_is_checked():
    """Every kernel configuration (f16_key) a supported fp16 plan reaches is reached by an exactly checked plan."""
    have = {}
    for plan in CHECKED_F16:
        for k, where in _plan_keys(plan).items():
            have.setdefault(k, where)
    missing = {}
    for plan in SUPPORTED_F16:
        for k, where in _plan_keys(plan).items():
            if k not in have:
                missing.setdefault(k, where)
    print(f"{len(have)} fp16 configuration keys over the checked plans")
    for k, where in missing.items():
        print(f"MISSING {k}: {where}")
    assert not missing, f"{len(missing)} fp16 configurations no exact check runs: " + "; ".join(
        f"{k} ({w})" for k, w in missing.items())


def test_decode_of_the_plans_own_logits_bit_for_bit_with_ties(calibrated):
    """A calibrated yolov5s, half; anchor 0 of every level gets theta biases of 9..12.5, where ATen's half sigmoid rounds to
    1.0: its rows' first maximum over the fp16 sigmoids is then bin 0 while the logits' maximum lies elsewhere."""
    m = copy.deepcopy(calibrated).half()
    det = m.model[-1]
    with torch.no_grad():
        for mi in det.m:
            b = mi.bias.view(det.na, det.no)
            b[0, 5 + det.nc:] = torch.arange(180, dtype=torch.float32).remainder(15).mul(0.25).add(9.0).half()
    m = m.to(DEV)
    x = synth_tiles(2, 512, seed=3).to(DEV)
    st = _stats()
    for compact in (False, True):
        eng = InferenceEngine(m, 2, 512, 512, DEV, compact_detect=compact)
        eng.forward(x)
        raw = torch.empty(eng.pred.shape[:2] + (eng.no,), dtype=torch.float16, device=DEV)
        for op in eng.convs:
            if op.desc.mode == MODE_DETECT:
                check_detect(op, raw, st, f"calibrated {'records' if compact else 'eval'}", integer=False)
    print(st)
    assert st["theta_moved"] > 1000   # rows whose fp16-sigmoid first maximum is not the logits' arg-max


def test_half_threshold_is_torchs_half_comparison():
    v = torch.linspace(0, 0.01, 20001, dtype=torch.float32)
    vh = v.half()
    for thr in (0.001, 0.01, 0.1, 0.25, 0.3, 0.45, 1 / 3):
        got = (vh.to(DEV) > thr).cpu()
        assert torch.equal(got, vh.float() > half_threshold(thr)), thr
        assert torch.equal((vh.to(DEV) > thr).cpu(), (vh.float().to(DEV) > half_threshold(thr)).cpu())
    assert half_threshold(0.001) == float(np.float16(0.001)) and half_threshold(0.001) != 0.001


def _oracle_half_nms(pred16, conf_thres, iou_thres, multi_label, max_det):
    """oracle/postprocess.py on the fp16 rows with general.py:797/:820/:830's half arithmetic: the conf filter and product
    are evaluated on the half tensor here (obj = 1 keeps the oracle's own product exact)."""
    thr = half_threshold(conf_thres)
    p = pred16.clone()
    keep = p[..., 4:5] > conf_thres                         # torch's half comparison
    conf = p[..., 5:5 + 15] * p[..., 4:5]                   # half product
    conf = torch.where(conf.float() > thr, conf, torch.zeros_like(conf))
    p[..., 5:5 + 15] = conf
    p[..., 4:5] = keep.half()
    return oracle_nms(p.float(), conf_thres, iou_thres, multi_label=multi_label, max_det=max_det)


@pytest.mark.parametrize("multi_label", [False, True])
def test_records_nms_equals_oracle_on_half_rows(calibrated, multi_label):
    m = copy.deepcopy(calibrated).half().to(DEV)
    x = synth_tiles(2, 1024, seed=5).to(DEV)
    rows = m(x)[0].clone()
    rec = m.detect_records(x)
    assert isinstance(rec, DetectRecords) and rec.half and rows.dtype == torch.float16
    got = non_max_suppression_obb(rec, 0.25, 0.45, multi_label=multi_label, max_det=1500)
    # the raw-tensor route on the rows with the half conf filter and product applied (obj = 1): the same detections
    p = rows.clone()
    keep = p[..., 4:5] > 0.25
    conf = p[..., 5:5 + 15] * p[..., 4:5]
    p[..., 5:5 + 15] = torch.where(conf.float() > half_threshold(0.25), conf, torch.zeros_like(conf))
    p[..., 4:5] = keep.half()
    raw = non_max_suppression_obb(p.float(), 0.25, 0.45, multi_label=multi_label, max_det=1500)
    for g, r in zip(got, raw):
        assert torch.equal(g, r)
    if not multi_label:
        return
    want = _oracle_half_nms(rows, 0.25, 0.45, multi_label, 1500)
    n = 0
    for g, w in zip(got, want):   # the same rows; fp16 scores tie often, and tied rows may come in another order
        g = g.cpu()
        assert g.shape == w.shape, (g.shape, w.shape)
        assert torch.equal(g[:, 5], w[:, 5].to(g.dtype)), "scores"
        order = lambda t: t[np.lexsort(t.numpy().T[::-1])]   # noqa: E731
        assert torch.equal(order(g), order(w.to(g.dtype)))
        n += g.shape[0]
    assert n > 50


def _s2d16(img, Hp, Wp):
    """[B, 3, Hp, Wp] fp16 -> the stem layout [B, Hp/2, Wp/2 + 2, 16] fp16 (pad pixels and channels 12-15 zero)."""
    B = img.shape[0]
    xs = torch.zeros((B, Hp // 2, Wp // 2 + 2, 16), dtype=torch.float16, device=DEV)
    for dy in range(2):
        for dx in range(2):
            xs[:, :, 1:-1, (dy * 2 + dx) * 3:(dy * 2 + dx) * 3 + 3] = img[:, :, dy::2, dx::2].permute(0, 2, 3, 1)
    return xs


def test_stem_and_tta_resample_bit_for_bit():
    m = half_mirror("n")
    B, H, W = 2, 256, 320
    u8 = torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, device=DEV)
    f32 = torch.rand((B, 3, H, W), device=DEV)
    plan = TTAPlan(m, B, H, W, DEV)
    for x, img in ((u8, u8.half() / 255), (f32, f32.half())):   # val.py:187-188: im.half(), im /= 255
        plan.forward(x)
        torch.cuda.synchronize()
        assert torch.equal(bits(plan.engines[0].x_s2d), bits(_s2d16(img, H, W))), f"stem {x.dtype}"
        for k in (1, 2):
            g = plan.branches[k]
            src = img.flip(3) if g["flip"] == 3 else img
            r = F.interpolate(src, size=(g["h"], g["w"]), mode="bilinear", align_corners=False)
            r = F.pad(r, [0, g["Wp"] - g["w"], 0, g["Hp"] - g["h"]], value=0.447)
            got = plan.engines[k].x_s2d
            assert torch.equal(bits(got), bits(_s2d16(r, g["Hp"], g["Wp"]))), f"resample branch {k} {x.dtype}"


def _dist(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


def test_plan_distance_from_fp32(calibrated):
    """The fp16 plan's Detect rows are closer to the fp32 eager forward than the bf16 plan's, and within
    HALF_EAGER_MULTIPLE x torch's own half forward's distance (calibrated yolov5s, uint8 tiles)."""
    m = copy.deepcopy(calibrated)
    x = synth_tiles(2, 1024, seed=7).to(DEV)
    xf = x.float() / 255
    ref = EagerFusedModel(m, DEV, half=False).forward(xf).float()
    eager16 = EagerFusedModel(m, DEV, half=True).forward(x.half() / 255).float()
    md = m.to(DEV)
    bf = md(x)[0].float().clone()
    md.half()
    fp = md(x)[0].float()
    cols = slice(0, 5 + 15)
    d_bf, d_fp, d_eager = (_dist(t[..., cols], ref[..., cols]) for t in (bf, fp, eager16))
    print(f"relative L2 distance from fp32 (box, obj, cls): bf16 plan {d_bf:.3e}, fp16 plan {d_fp:.3e}, "
          f"torch half eager {d_eager:.3e}, ratio {d_fp / d_eager:.2f}")
    assert d_fp < d_bf
    assert d_fp <= HALF_EAGER_MULTIPLE * d_eager


def test_half_model_through_pipeline_and_scene(calibrated):
    from yolov5_obb_b200.pipeline import DetectPipeline
    from yolov5_obb_b200.scene import SceneDetector
    m = copy.deepcopy(calibrated).half().to(DEV)
    imgs = [synth_tiles(1, 640, seed=s)[0].permute(1, 2, 0).contiguous().numpy() for s in (1, 2)]
    pipe = DetectPipeline(m, 0.25, 0.45, 300, multi_label=True, device=DEV)
    outs = list(pipe.run_images(imgs, img_size=640))
    assert len(outs) == 2
    eng = m.records_plan((1, 3, 640, 640), DEV)
    assert eng.half and eng.x_s2d.dtype == torch.float16
    scene = synth_tiles(1, 1500, seed=4)[0].permute(1, 2, 0).contiguous().to(DEV)
    res = SceneDetector(m, batch_size=2).det(scene)
    assert res.rows.shape[0] > 0 and torch.isfinite(res.rows).all()


def _u8_of(x16):
    """The uint8 samples an fp16 stem input holds (fp16(u * (1 / 255)) is one-to-one on 0..255)."""
    u = (x16.float() * 255).round()
    assert ((u >= 0) & (u <= 255)).all()
    return u


def test_letterbox_and_scene_tiles_bit_for_bit():
    """The fp16 letterbox and scene-tile staging: torch's `u8.half() / 255` of the very samples the bf16 kernels stage
    (those are checked against cv2 and the tile crop in tests/test_letterbox_gpu.py and tests/test_scene_gpu.py)."""
    from tests.test_scene_gpu import _scene, _torch_tiles
    from yolov5_obb_b200 import _lib
    from yolov5_obb_b200 import letterbox as P
    from yolov5_obb_b200.scene import split_origins, tile_geometry
    rng = np.random.default_rng(0)
    images = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in ((700, 900), (512, 300))]
    Hp = Wp = 640
    places = [P.place_detect(im.shape[0], im.shape[1], 640, auto=False)[0] for im in images]
    batch = P.pack_batch(images, places, Hp, Wp)
    dev = batch.host[:batch.nbytes].to(DEV)
    xs = {dt: torch.zeros((2, Hp // 2, Wp // 2 + 2, 16), dtype=dt, device=DEV) for dt in (torch.bfloat16, torch.float16)}
    for x in xs.values():
        P.letterbox_s2d(dev, batch, x, 1)
    torch.cuda.synchronize()
    u = _u8_of(xs[torch.float16])
    assert torch.equal(bits(xs[torch.float16]), bits(u.half() / 255)), "letterbox fp16"
    assert torch.equal(bits(xs[torch.bfloat16]), bits((u / 255).bfloat16())), "letterbox: not the bf16 kernel's samples"

    H, W = 1700, 2300
    scene = _scene(H, W, 1)
    origins = split_origins(H, W)
    size, border, _ = tile_geometry(1024, 0.5)
    T = len(origins)
    got = torch.zeros((T, size // 2, size // 2 + 2, 16), dtype=torch.float16, device=DEV)
    org = torch.tensor(origins, dtype=torch.int32, device=DEV)
    sd = scene.to(DEV)
    _lib.check(_lib.lib().y5obb_scene_tiles_s2d_u8_f16(sd.data_ptr(), H, W, org.data_ptr(), T, 1024, size, border,
                                                       got.data_ptr(), 1, _lib.stream_ptr(torch.device(DEV))), "scene f16")
    tiles = _torch_tiles(scene, origins, 1024, size, border).to(DEV)
    assert torch.equal(bits(got), bits(_s2d16(tiles.half() / 255, size, size))), "scene tiles fp16"


def _integer_head(plan, seed):
    """Overwrites the plan's Detect inputs and head operands with multiples of 1/8 (features, weights) and 1/32 (bias, up to
    +-48): every logit is exact in fp32 in any summation order, and those above 32 in magnitude round to fp16.  -> the logits
    [B, na, H, W, no] the half Detect conv would output, as fp32."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for x, w, b in plan.head_inputs():
        x.view().copy_(torch.randint(-16, 17, x.view().shape, generator=g, device=DEV).half() / 8)
        wv = torch.randint(-8, 9, w.shape, generator=g, device=DEV) * (torch.rand(w.shape, generator=g, device=DEV) < 0.05)
        w.copy_(wv.half() / 8)
        b.copy_(torch.randint(-1536, 1537, b.shape, generator=g, device=DEV).float() / 32)
        lg = x.view().double() @ w.double().t() + b.double()
        B, H, W = x.B, x.H, x.W
        na = plan.na
        out.append(lg.float().half().float().view(B, H, W, na, plan.no).permute(0, 3, 1, 2, 4).contiguous())
    return out


def test_fp16_validation_loss_bit_for_bit():
    """ComputeLoss.head_items on an fp16 plan equals ComputeLoss on the fp16-rounded logits (val.py:198-199's
    `compute_loss([x.float() for x in train_out])` of a half model), bit for bit."""
    from tests import vallossgen as VG
    from yolov5_obb_b200.loss import ComputeLoss
    m = build_mirror("s", nc=15, seed=0, obj_bias=VG.OBJ_BIAS).half().to(DEV)
    m.hyp = loss_ref.scaled_hyp(loss_ref.DEFAULT_HYP, 3, 15, VG.HYP_IMGSZ)
    cl = ComputeLoss(m)
    n_round = 0
    for i in range(2):
        im, tg = VG.batch(i)
        m.detect_records(im.to(DEV))
        plan = m.records_plan(tuple(im.shape), DEV)
        p = _integer_head(plan, i)
        n_round += sum(int((t.abs() > 32).sum()) for t in p)
        loss, items = cl.head_items(plan, tg.to(DEV))
        want_loss, want_items = cl(p, tg.to(DEV))
        torch.cuda.synchronize()
        assert torch.equal(bits(items), bits(want_items.float())), (items, want_items)
        assert torch.equal(bits(loss), bits(want_loss.float().reshape(loss.shape))), (loss, want_loss)
    assert n_round > 1000


def test_half_validator_with_loss():
    """Validator on a half model, with and without compute_loss: the same mAP, and the loss of the per-batch head_items."""
    from tests.test_valloss_gpu import _assert_validator, _validator_setup
    model, batches, loader_fn = _validator_setup()
    loader = loader_fn(model, batches, 0.1)
    model.half()
    v = _assert_validator(model, loader, conf_thres=0.1, iou_thres=0.4, max_det=300)
    assert model.records_plan(tuple(loader[0][0].shape), DEV).half and v is not None
