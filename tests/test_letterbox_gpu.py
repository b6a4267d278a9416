"""GPU tests of the image front end (yolov5_obb_b200/letterbox.py, csrc/letterbox.cu): the letterbox kernel's stem input
against y5obb_stem_s2d_u8 applied to the CPU restatement's letterboxed batch (oracle/letterbox_ref.py, pinned against cv2 and
the reference in tests/test_letterbox_cpu.py) and to the reference's own bytes (letterbox_golden.npz), bit for bit; the batched
polygon kernel against rbox2poly + scale_polys per image; DetectPipeline.run_images and the Validator's raw form against the
existing tensor paths fed the restatement's images; and the refusals."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import letterbox_ref as R
from tests import letterboxgen as LG
from yolov5_obb_b200 import _lib
from yolov5_obb_b200 import letterbox as P

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
G = np.load(Path(__file__).resolve().parent / "golden" / "letterbox_golden.npz")
S = LG.GOLDEN_IMG_SIZE
SENTINEL = 0x7BCD   # a bf16 bit pattern no pixel produces


def _kernel(images, places, Hp, Wp, pad_cols=2):
    """y5obb_letterbox_s2d_u8 into the middle of a sentinel-filled buffer -> (whole buffer as int16, the batch's slice)."""
    B = len(images)
    batch = P.pack_batch(images, places, Hp, Wp)
    dev = batch.host[:batch.nbytes].to(DEV)
    n = B * (Hp // 2) * (Wp // 2 + 2 * pad_cols) * 16
    guard = 4096
    raw = torch.full((n + 2 * guard,), SENTINEL, dtype=torch.int16, device=DEV)
    x = raw[guard:guard + n].view(torch.bfloat16).view(B, Hp // 2, Wp // 2 + 2 * pad_cols, 16)
    P.letterbox_s2d(dev, batch, x, pad_cols)
    torch.cuda.synchronize()
    return raw, guard, n


def _stem(nchw_u8, pad_cols=2):
    B, _, Hp, Wp = nchw_u8.shape
    n = B * (Hp // 2) * (Wp // 2 + 2 * pad_cols) * 16
    guard = 4096
    raw = torch.full((n + 2 * guard,), SENTINEL, dtype=torch.int16, device=DEV)
    x = torch.from_numpy(np.ascontiguousarray(nchw_u8)).to(DEV)
    _lib.check(_lib.lib().y5obb_stem_s2d_u8(x.data_ptr(), raw[guard:].data_ptr(), B, Hp, Wp, pad_cols,
                                            _lib.stream_ptr(torch.device(DEV))), "y5obb_stem_s2d_u8")
    torch.cuda.synchronize()
    return raw


def _oracle_rect(images, img_size, batch_shape):
    return np.stack([R.rect_item(im, img_size, batch_shape)[0] for im in images])


def _check(images, places, Hp, Wp, want_nchw):
    got, guard, n = _kernel(images, places, Hp, Wp)
    want = _stem(want_nchw)
    assert torch.equal(got, want)   # pixels, the untouched pad columns and the guards on both sides
    assert int((got[guard:guard + n] == SENTINEL).sum()) == len(images) * (Hp // 2) * 4 * 16


@pytest.mark.parametrize("B", [1, 16])
def test_rect_batches_equal_stem_of_oracle(B):
    """Mixed sizes and modes in one launch: fractional INTER_AREA, integer blocks (2x, 3x, 4x), no resize, INTER_LINEAR
    enlargement - whatever load_image_label chooses for each image."""
    sizes = (LG.GOLDEN_SIZES + [(200, 320), (512, 512), (77, 300), (1024, 999), (131, 640)])[:B]
    images = [LG.synth_image(h, w, 40 + i) for i, (h, w) in enumerate(sizes)]
    img_size = 256
    _, shapes = P.rect_batch_shapes([(w, h) for h, w in sizes], B, img_size, 32, 0.5)
    Hp, Wp = int(shapes[0][0]), int(shapes[0][1])
    places = [P.place_rect(h, w, img_size, (Hp, Wp)) for h, w in sizes]
    if B == 16:
        modes = {P.resample_plan(p.h0, p.w0, p.new_h, p.new_w, p.interp)[0] for p in places}
        assert modes == {P.MODE_COPY, P.MODE_LINEAR, P.MODE_AREA_INT, P.MODE_AREA}
    _check(images, places, Hp, Wp, _oracle_rect(images, img_size, (Hp, Wp)))


@pytest.mark.parametrize("h0,w0,img_size", [(1689, 2425, 1024), (4000, 4000, 1024), (2048, 2048, 1024), (800, 1333, 1024),
                                            (300, 500, 1024), (3000, 1000, 640), (1024, 1024, 1024)])
def test_detect_letterbox_equals_stem_of_oracle(h0, w0, img_size):
    """detect.py's letterbox (INTER_LINEAR, the exact-2x switch to INTER_AREA, enlargement, minimum rectangle)."""
    im = LG.synth_image(h0, w0, h0 + w0)
    p, (Hp, Wp) = P.place_detect(h0, w0, img_size, 32, True)
    want = R.to_chw_rgb(R.letterbox(im, img_size, auto=True, stride=32)[0])[None]
    assert want.shape[2:] == (Hp, Wp)
    _check([im], [p], Hp, Wp, want)


def test_area_4000_batch_equals_stem_of_oracle():
    """Large sources through load_image_label's INTER_AREA: 4000^2 -> 1024^2 (fractional) and 4096 x 2048 (exact 4x)."""
    images = [LG.synth_image(4000, 4000, 1), LG.synth_image(4096, 2048, 2)]
    places = [P.place_rect(im.shape[0], im.shape[1], 1024, (1024, 1024)) for im in images]
    _check(images, places, 1024, 1024, _oracle_rect(images, 1024, (1024, 1024)))


def test_golden_cases_equal_reference_bytes():
    """The reference's own LoadImages / LoadImagesAndLabels bytes on the seeded images (the subset the golden keeps in full)."""
    images = LG.golden_images()
    for i in LG.GOLDEN_FULL_DETECT:
        im = images[i]
        p, (Hp, Wp) = P.place_detect(im.shape[0], im.shape[1], S, 32, True)
        _check([im], [p], Hp, Wp, G[f"detect/auto1/{i}"][None])
    order, shapes = P.rect_batch_shapes([(w, h) for h, w in LG.GOLDEN_SIZES], LG.GOLDEN_BATCH, S, 32, LG.GOLDEN_PAD)
    for b in LG.GOLDEN_FULL_RECT_BATCHES:
        ks = [k for k in range(len(order)) if G["rect/batch"][k] == b]
        ims = [images[order[k]] for k in ks]
        Hp, Wp = int(shapes[b][0]), int(shapes[b][1])
        places = [P.place_rect(im.shape[0], im.shape[1], S, (Hp, Wp)) for im in ims]
        _check(ims, places, Hp, Wp, np.stack([G[f"rect/{k}/img"] for k in ks]))


def test_scale_polys_batched_equals_the_two_calls():
    from yolov5_obb_b200.rboxs_utils import rbox2poly, scale_polys
    g = torch.Generator().manual_seed(3)
    B, max_det = 5, 300
    rows = torch.rand((B, max_det, 7), generator=g) * torch.tensor([1024.0, 1024.0, 200.0, 60.0, 3.1, 1.0, 15.0])
    rows[..., 4] -= 1.55
    counts = torch.tensor([0, max_det, 17, 1, 299, 12345], dtype=torch.int64)   # (a trailing entry, as the async form has)
    pg = torch.tensor([[0.0, 11.5, 0.4222], [16.0, 16.0, 1.0], [3.5, 0.0, 1.7], [0.25, 0.75, 0.333], [12.0, 0.0, 0.256]])
    got = P.scale_polys_batched(rows.to(DEV), counts.to(DEV), pg.to(DEV)).cpu()
    for b in range(B):
        k = int(counts[b])
        want = rbox2poly(rows[b, :k, :5].contiguous().to(DEV))
        if k:
            scale_polys(None, want, None, ratio_pad=((float(pg[b, 2]), float(pg[b, 2])), (float(pg[b, 0]), float(pg[b, 1]))))
        assert torch.equal(got[b, :k], want.cpu().reshape(k, 8))
        assert not got[b, k:].any()


@pytest.fixture(scope="module")
def model():
    from tests.modelgen import build_mirror
    from yolov5_obb_b200 import general
    m = build_mirror("n", nc=15, seed=0, obj_bias=1.0, cls_bias=-1.0, det_gain=6.0).to(DEV)
    yield m
    # these tests plan many input shapes on several pipelines' streams: release the plans, the post-process graphs and the
    # per-stream workspaces with the module instead of leaving them resident for the rest of the session
    m._engines.clear()
    general._GRAPHS.clear()
    _lib._WS.clear()
    torch.cuda.empty_cache()


KW = dict(conf_thres=0.25, iou_thres=0.45, max_det=300)
E2E_SIZES = [(300, 400), (256, 256), (97, 211), (512, 512), (384, 384), (200, 140), (128, 128), (260, 250), (640, 333)]


def _existing_path(model, nchw_u8, pad_gains):
    """The existing calls on letterboxed tensors: detect_records + non_max_suppression_obb, rbox2poly + scale_polys per image."""
    from yolov5_obb_b200.general import non_max_suppression_obb
    from yolov5_obb_b200.rboxs_utils import rbox2poly, scale_polys
    x = torch.from_numpy(np.ascontiguousarray(nchw_u8)).to(DEV)
    dets = non_max_suppression_obb(model.detect_records(x), multi_label=True, **KW)
    out = []
    for d, (px, py, gain) in zip(dets, pad_gains):
        d = d.clone()
        poly = rbox2poly(d[:, :5].contiguous())
        if d.shape[0]:
            scale_polys(None, poly, None, ratio_pad=((gain, gain), (px, py)))
        out.append((poly.reshape(-1, 8).cpu(), d.cpu()))
    return out


@pytest.mark.parametrize("slots", [1, 2])
def test_run_images_detect_mode_equals_existing_path(model, slots):
    from yolov5_obb_b200.pipeline import DetectPipeline
    images = [LG.synth_image(h, w, 70 + i) for i, (h, w) in enumerate(E2E_SIZES)]
    img_size = 256
    want = []
    for im in images:
        lbx = R.to_chw_rgb(R.letterbox(im, img_size, auto=True, stride=32)[0])[None]
        want += _existing_path(model, lbx, [P.detect_pad_gain(lbx.shape[2:], im.shape[:2])])
    pipe = DetectPipeline(model, multi_label=True, device=DEV, slots=slots, **KW)
    got = list(pipe.run_images(iter(images), img_size=img_size, stride=32, auto=True))
    assert len(got) == len(images) and sum(w[1].shape[0] for w in want) > 50
    for g, (poly, rows), im in zip(got, want, images):
        assert torch.equal(g.rows, rows) and torch.equal(g.polys, poly)
        assert torch.equal(g.conf, rows[:, 5]) and torch.equal(g.cls, rows[:, 6]) and g.shapes[0] == im.shape[:2]
    assert [torch.equal(a.rows, b.rows) for a, b in zip(pipe.run_images(images, img_size=img_size), got)] == [True] * len(images)


@pytest.mark.parametrize("slots", [1, 2])
def test_run_images_rect_mode_equals_existing_path(model, slots):
    from yolov5_obb_b200.pipeline import DetectPipeline
    images = [LG.synth_image(h, w, 70 + i) for i, (h, w) in enumerate(E2E_SIZES)]
    img_size, bs = 256, 2
    order, shapes = R.rect_batch_shapes([(im.shape[1], im.shape[0]) for im in images], bs, img_size, 32, 0.5)[::2]
    want = [None] * len(images)
    for b in range(len(shapes)):
        idx = [int(k) for k in order[b * bs:(b + 1) * bs]]
        items = [R.rect_item(images[k], img_size, shapes[b]) for k in idx]
        res = _existing_path(model, np.stack([it[0] for it in items]),
                             [(it[1][1][1][0], it[1][1][1][1], it[1][1][0][0]) for it in items])
        for k, r in zip(idx, res):
            want[k] = r
    pipe = DetectPipeline(model, multi_label=True, device=DEV, slots=slots, **KW)
    got = list(pipe.run_images(images, img_size=img_size, stride=32, auto=False, batch_size=bs, pad=0.5))
    assert len(got) == len(images) and sum(w[1].shape[0] for w in want) > 50
    for g, (poly, rows) in zip(got, want):
        assert torch.equal(g.rows, rows) and torch.equal(g.polys, poly)


def test_validator_raw_form_equals_tensor_form(model):
    from yolov5_obb_b200.rboxs_utils import poly2rbox
    from yolov5_obb_b200.val import Validator
    images = [LG.synth_image(h, w, 70 + i) for i, (h, w) in enumerate(E2E_SIZES)]
    img_size, bs = 256, 3
    order, shapes = P.rect_batch_shapes([(im.shape[1], im.shape[0]) for im in images], bs, img_size, 32, 0.5)
    raw, tens = [], []
    for b in range(len(shapes)):
        idx = [int(k) for k in order[b * bs:(b + 1) * bs]]
        places = [P.place_rect(images[k].shape[0], images[k].shape[1], img_size, shapes[b]) for k in idx]
        tg = []
        for j, (k, p) in enumerate(zip(idx, places)):
            polys = p.map_labels(LG.synth_polys(images[k].shape[0], images[k].shape[1], 4, 900 + k))
            rb = poly2rbox(torch.from_numpy(polys).float().to(DEV), use_pi=True).float().cpu()
            tg.append(torch.cat([torch.full((4, 1), float(j)), torch.full((4, 1), float(k % 15)), rb], 1))
        targets = torch.cat(tg)
        sh = [p.shapes for p in places]
        raw.append(([images[k] for k in idx], targets, None, sh))
        tens.append((torch.from_numpy(_oracle_rect([images[k] for k in idx], img_size, shapes[b])), targets, None, sh))
    a = Validator(model, max_det=300)(raw)
    b = Validator(model, max_det=300)(tens)
    assert a.seen == b.seen == len(images)
    assert a.results == b.results and np.array_equal(a.maps, b.maps) and np.array_equal(a.nt, b.nt)
    assert np.array_equal(a.ap_full, b.ap_full) and np.array_equal(a.p_curve, b.p_curve)
    with pytest.raises(RuntimeError):
        Validator(model, augment=True)([raw[0]])
    with pytest.raises(RuntimeError):
        Validator(model)([(raw[0][0][:1], raw[0][1], None, raw[0][3])])


def test_refusals(model):
    from yolov5_obb_b200.pipeline import DetectPipeline
    pipe = DetectPipeline(model, device=DEV, **KW)
    ok = LG.synth_image(64, 64, 0)
    for bad in (ok.astype(np.float32), ok[:, :, :2], ok.transpose(2, 0, 1), np.zeros((0, 64, 3), np.uint8),
                torch.from_numpy(ok).to(DEV)):
        with pytest.raises(RuntimeError):
            list(pipe.run_images([bad], img_size=128))
    with pytest.raises(RuntimeError, match="multiple"):
        list(pipe.run_images([ok], img_size=100))
    with pytest.raises(RuntimeError, match="multiple"):
        list(pipe.run_images([ok], img_size=128, stride=16))
    with pytest.raises(RuntimeError):
        list(pipe.run_images([ok], img_size=128, auto=True, batch_size=2))
    with pytest.raises(RuntimeError):
        list(DetectPipeline(model, device=DEV, fused_detect=False, **KW).run_images([ok], img_size=128))
    assert list(pipe.run_images([], img_size=128)) == [] and list(pipe.run_images([], img_size=128, auto=False)) == []
    # the C entry refuses descriptors that reach outside the source buffer, the tables or the letterboxed image
    p, (Hp, Wp) = P.place_detect(64, 64, 128, 32, True)
    batch = P.pack_batch([ok], [p], Hp, Wp)
    x = torch.zeros((1, Hp // 2, Wp // 2 + 2, 16), dtype=torch.bfloat16, device=DEV)
    w32 = batch.host.numpy()[:batch.desc_bytes].view(np.int32)
    for word, value in ((2, 65), (6, Hp), (8, 7), (12, 1 << 28), (0, 1 << 20)):
        keep = int(w32[word])
        w32[word] = value
        with pytest.raises(RuntimeError, match="EINVAL"):
            P.letterbox_s2d(batch.host[:batch.nbytes].to(DEV), batch, x, 1)
        w32[word] = keep
    P.letterbox_s2d(batch.host[:batch.nbytes].to(DEV), batch, x, 1)
    with pytest.raises(RuntimeError):
        P.letterbox_s2d(batch.host[:batch.nbytes].to(DEV), batch, x[:, :, :-1], 1)
