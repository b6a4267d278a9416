"""CPU: the numpy restatement of the image front end (oracle/letterbox_ref.py) against the installed cv2 over a sweep of size
pairs and against the REFERENCE's own letterbox / LoadImages / LoadImagesAndLabels(rect=True) outputs
(tests/golden/letterbox_golden.npz); and the host geometry, coefficient tables and batch packing of
yolov5_obb_b200/letterbox.py against both."""
import hashlib
from pathlib import Path

import numpy as np
import pytest

from oracle import letterbox_ref as R
from tests import letterboxgen as LG
from yolov5_obb_b200 import letterbox as P

G = np.load(Path(__file__).resolve().parent / "golden" / "letterbox_golden.npz")
S = LG.GOLDEN_IMG_SIZE


def _pairs():
    """(source (h, w), destination (h, w)) pairs: one-pixel-off sizes, exact 2x / 3x / 4x, odd sizes, extreme aspect ratios,
    then seeded random ones; enlargements included (INTER_LINEAR only uses them)."""
    fixed = [((64, 64), (32, 32)), ((65, 64), (33, 31)), ((100, 37), (99, 38)), ((37, 100), (64, 173)), ((512, 512), (256, 256)),
             ((300, 200), (150, 100)), ((300, 200), (150, 101)), ((10, 500), (7, 333)), ((500, 10), (999, 20)),
             ((1, 50), (1, 25)), ((50, 1), (100, 3)), ((333, 777), (1024, 439)), ((129, 257), (64, 128)), ((90, 90), (30, 30)),
             ((90, 90), (31, 30)), ((96, 60), (24, 20)), ((96, 60), (24, 30)), ((400, 400), (100, 100)), ((401, 400), (100, 100)),
             ((60, 60), (60, 20)), ((60, 60), (59, 60)), ((7, 7), (1, 1)), ((9, 12), (3, 4)), ((500, 500), (167, 167)),
             ((101, 77), (100, 76)), ((2, 2), (1, 1)), ((1689, 2425), (713, 1024)), ((800, 1333), (615, 1024)),
             ((2048, 2048), (1024, 1024)), ((3072, 96), (1024, 32)), ((4096, 64), (1024, 16)), ((64, 4096), (16, 1024)),
             ((4096, 33), (1000, 8)), ((1025, 1023), (1024, 1022)), ((3, 3), (11, 5)), ((7, 9), (21, 27))]
    rng = np.random.default_rng(7)
    rand = []
    for _ in range(180):
        h0, w0 = (int(v) for v in rng.integers(1, 600, 2))
        rand.append(((h0, w0), (int(rng.integers(1, 700)), int(rng.integers(1, 700)))))
    return fixed + rand


PAIRS = _pairs()


def test_resamplers_equal_installed_cv2():
    cv2 = pytest.importorskip("cv2")
    assert len(PAIRS) >= 200
    rng = np.random.default_rng(0)
    n_lin = n_area = n_two = 0
    for (h0, w0), (h, w) in PAIRS:
        im = rng.integers(0, 256, (h0, w0, 3), dtype=np.uint8)
        want = cv2.resize(im, (w, h), interpolation=cv2.INTER_LINEAR)
        assert np.array_equal(R.resize(im, (w, h), R.LINEAR), want), ("linear", h0, w0, h, w)
        n_lin += 1
        n_two += (h0 == 2 * h and w0 == 2 * w)
        hs, ws = min(h, h0), min(w, w0)   # INTER_AREA: shrinking only
        want = cv2.resize(im, (ws, hs), interpolation=cv2.INTER_AREA)
        assert np.array_equal(R.resize(im, (ws, hs), R.AREA), want), ("area", h0, w0, hs, ws)
        n_area += 1
    assert n_lin >= 200 and n_area >= 200 and n_two >= 3


def test_exact_2x_linear_is_area():
    im = LG.synth_image(512, 512, 1)
    assert np.array_equal(R.resize(im, (256, 256), R.LINEAR), R.resize(im, (256, 256), R.AREA))
    assert P.resample_plan(512, 512, 256, 256, P.LINEAR)[0] == P.MODE_AREA_INT
    assert P.resample_plan(512, 512, 256, 255, P.LINEAR)[0] == P.MODE_LINEAR
    assert P.resample_plan(384, 384, 128, 128, P.AREA)[:3] == (P.MODE_AREA_INT, 3, 3)
    assert P.resample_plan(300, 400, 96, 128, P.AREA)[0] == P.MODE_AREA
    assert P.resample_plan(128, 128, 128, 128, P.AREA)[0] == P.MODE_COPY
    with pytest.raises(RuntimeError):
        P.resample_plan(100, 100, 128, 128, P.AREA)
    with pytest.raises(RuntimeError):
        P.resample_plan(100, 100, 50, 50, "cubic")


def test_geometry_equals_reference_letterbox():
    g = G["geometry"]
    assert g.shape[0] >= 800
    for row in g:
        h0, w0, nh, nw = (int(v) for v in row[:4])
        auto, fill, up, stride = bool(row[4]), bool(row[5]), bool(row[6]), int(row[7])
        for mod in (P, R):
            unpad, border, ratio, pad = mod.letterbox_geometry((h0, w0), (nh, nw), auto, fill, up, stride)
            if row[8] >= 0:
                assert tuple(unpad) == (int(row[8]), int(row[9]))
            else:   # the reference did not resize: new_unpad is the source size
                assert tuple(unpad) == (w0, h0)
            assert tuple(border) == tuple(int(v) for v in row[10:14])
            assert (ratio[0], ratio[1], float(pad[0]), float(pad[1])) == tuple(row[14:18])


def _same_bytes(got, key):
    """The golden keeps this image as shape + SHA-256 of its bytes."""
    return got.shape == tuple(G[key + "/shape"]) and \
        hashlib.sha256(np.ascontiguousarray(got).tobytes()).hexdigest() == str(G[key + "/sha256"])


def test_oracle_equals_reference_loaders_on_seeded_images():
    images = LG.golden_images()
    for i, im in enumerate(images):
        for auto in (True, False):
            assert _same_bytes(R.to_chw_rgb(R.letterbox(im, S, auto=auto, stride=32)[0]), f"detect/auto{int(auto)}/{i}"), (auto, i)
        if i in LG.GOLDEN_FULL_DETECT:
            assert _same_bytes(G[f"detect/auto1/{i}"], f"detect/auto1/{i}")
    for i in (0, 2, 6):
        for new, auto, fill, up in ((S, False, True, True), ((96, 160), False, False, False), (160, True, False, True)):
            got = R.letterbox(images[i], new, auto=auto, scaleFill=fill, scaleup=up, stride=32)[0]
            assert _same_bytes(got, f"lb/{i}/{new}/{int(auto)}{int(fill)}{int(up)}")


def _rect(mod):
    shapes_wh = [(w, h) for h, w in LG.GOLDEN_SIZES]
    out = mod.rect_batch_shapes(shapes_wh, LG.GOLDEN_BATCH, S, 32, LG.GOLDEN_PAD)
    return out[0], out[-1]


def test_rect_loader_equals_reference():
    images = LG.golden_images()
    for mod in (P, R):
        order, shapes = _rect(mod)
        assert np.array_equal(order, G["rect/order"])
        assert np.array_equal(shapes, G["rect/batch_shapes"])
    order, shapes = _rect(P)
    for k, i in enumerate(order):
        bs = shapes[G["rect/batch"][k]]
        img, entry, _, _ = R.rect_item(images[i], S, bs)
        assert _same_bytes(img, f"rect/{k}"), k
        if G["rect/batch"][k] in LG.GOLDEN_FULL_RECT_BATCHES:
            assert np.array_equal(img, G[f"rect/{k}/img"]), k
        want = G[f"rect/{k}/shapes"]
        flat = lambda e: (e[0][0], e[0][1], e[1][0][0], e[1][0][1], float(e[1][1][0]), float(e[1][1][1]))
        assert flat(entry) == tuple(want)
        h0, w0 = images[i].shape[:2]
        p = P.place_rect(h0, w0, S, bs)
        assert flat(p.shapes) == tuple(want)
        q, hw = P.place_from_shapes(p.shapes)
        assert hw == tuple(int(v) for v in bs)
        assert (q.new_h, q.new_w, q.top, q.left, q.interp if (q.new_h, q.new_w) != (h0, w0) else None) == \
            (p.new_h, p.new_w, p.top, p.left, p.interp if (p.new_h, p.new_w) != (h0, w0) else None)
        rb = G[f"rect/{k}/rboxes"]
        if rb.shape[0] == 3:   # no label was filtered: the box centres are the mapped polygons' centres
            polys = np.array([[float(f"{v:.3f}") for v in row] for row in LG.synth_polys(h0, w0, 3, 500 + int(i))], np.float32)
            m = p.map_labels(polys)
            c = np.stack([m[:, 0::2].mean(1), m[:, 1::2].mean(1)], 1)
            assert np.abs(np.sort(c, 0) - np.sort(rb[:, 1:3].astype(np.float64), 0)).max() < 2e-2


def test_demo_image_equals_reference_loader():
    cv2 = pytest.importorskip("cv2")
    from oracle.build_ref import REF
    f = REF / "dataset" / "dataset_demo" / "images" / "P0032.png"
    if not f.exists():
        pytest.skip("the reference's demo image is not available")
    im = cv2.imread(str(f))
    for size in (256, 1024):
        assert tuple(im.shape[:2]) == tuple(G[f"demo/{size}/shape0"])
        assert _same_bytes(R.to_chw_rgb(R.letterbox(im, size, auto=True, stride=32)[0]), f"demo/{size}")


def _unpack(batch):
    """The packed buffer read back the way csrc/letterbox.cu reads it -> per image (descriptor words, source bytes)."""
    buf = batch.host.numpy()[:batch.nbytes]
    w32 = buf[:batch.desc_bytes].view(np.int32)
    out = []
    for b in range(batch.B):
        d = w32[16 * b:16 * b + 16]
        off = int(d[0:2].view(np.int64)[0])
        out.append((d, buf[batch.src_off + off:batch.src_off + off + int(d[2]) * int(d[3]) * 3].reshape(int(d[2]), int(d[3]), 3)))
    return w32, out


def test_pack_batch_layout_and_refusals():
    images = LG.golden_images()[:5]
    order, shapes = P.rect_batch_shapes([(im.shape[1], im.shape[0]) for im in images], 5, S, 32, 0.5)
    places = [P.place_rect(im.shape[0], im.shape[1], S, shapes[0]) for im in images]
    batch = P.pack_batch(images, places, int(shapes[0][0]), int(shapes[0][1]))
    w32, items = _unpack(batch)
    assert batch.src_off % 256 == 0 and batch.desc_bytes % 4 == 0
    for (d, src), im, p in zip(items, images, places):
        assert np.array_equal(src, im)
        assert tuple(d[2:8]) == (p.h0, p.w0, p.new_h, p.new_w, p.top, p.left)
        mode, kx, ky, inv, xt, yt = P.resample_plan(p.h0, p.w0, p.new_h, p.new_w, p.interp)
        assert d[8] == mode and d[12] % 2 == 0 and d[13] % 2 == 0
        assert np.array_equal(w32[d[12]:d[12] + xt.size], xt) and np.array_equal(w32[d[13]:d[13] + yt.size], yt)
    pg = batch.host.numpy()[batch.pad_gain_off:batch.pad_gain_off + 12 * batch.B].view(np.float32).reshape(-1, 3)
    assert np.array_equal(pg, np.array([p.pad_gain for p in places], np.float32))
    again = P.pack_batch(images, places, int(shapes[0][0]), int(shapes[0][1]), batch.host)
    assert again.host is batch.host
    for bad in (images[0].astype(np.float32), images[0][:, :, :2], images[0][:, :, 0], np.zeros((0, 5, 3), np.uint8), "x"):
        with pytest.raises(RuntimeError):
            P.as_image(bad)
    with pytest.raises(RuntimeError):
        P.pack_batch(images, places[:2], 128, 128)
    with pytest.raises(RuntimeError):
        P.place_rect(512, 300, S, (96, 96))   # a batch shape smaller than the resized image


def test_detect_pad_gain_is_scale_polys():
    p, (Hp, Wp) = P.place_detect(1689, 2425, 1024, 32, True)
    assert (Hp, Wp, p.new_h, p.new_w, p.top, p.left) == (736, 1024, 713, 1024, 11, 0)
    gain = min(Hp / 1689, Wp / 2425)
    assert p.pad_gain == ((Wp - 2425 * gain) / 2, (Hp - 1689 * gain) / 2, gain)
