"""Seeded synthetic loss inputs: Detect training outputs and DOTA-shaped targets with CSL rows
(targets[:, 7:] follow utils/rboxs_utils.py:9-26 gaussian_label_cpu, restated in numpy)."""
import numpy as np
import torch

PI = 3.141592


def gaussian_label(angle, num_class=180, sig=2.0):
    """utils/rboxs_utils.py:9-26 (u=0): peak at bin 90 - trunc(90 - angle)."""
    x = np.arange(-num_class / 2, num_class / 2)
    y = np.exp(-(x ** 2) / (2 * sig ** 2))
    index = int(num_class / 2 - angle)
    return np.concatenate([y[index:], y[:index]], axis=0)


def synth_targets(B, nt, imgsz, nc=15, seed=0):
    rng = np.random.default_rng(seed)
    t = np.zeros((nt, 187), np.float32)
    t[:, 0] = rng.integers(0, B, nt)
    t[:, 1] = rng.integers(0, nc, nt)
    t[:, 2:4] = rng.uniform(0, imgsz, (nt, 2))
    l = np.exp(rng.uniform(np.log(8), np.log(min(300, imgsz)), nt))
    t[:, 4] = l
    t[:, 5] = l * rng.uniform(0.15, 1.0, nt)
    k = rng.integers(0, 180, nt)
    theta = (k - 90) / 180 * PI
    t[:, 6] = theta
    for i in range(nt):
        angle = theta[i] * 180 / PI + 90
        t[i, 7:] = gaussian_label(angle)
    # duplicates: two targets in the same cell exercise the last-writer-wins tobj rule
    if nt >= 4:
        t[1, :] = t[0, :]
        t[1, 4:6] *= 1.1
        t[3, 2:4] = t[2, 2:4] + 0.5
    return t


def _f32_below(x):
    return float(np.nextafter(np.float32(x), np.float32(-np.inf)))


def _f32_above(x):
    return float(np.nextafter(np.float32(x), np.float32(np.inf)))


def boundary_targets(B, H, W, nc=15, seed=0):
    """[nt, 187] targets on build_targets' decision boundaries for an H x W input (strides 8, 16, 32, the default anchors), then
    12 random ones.  Every boundary centre is exact in fp32, and so is its quotient by each stride.  Image B - 1 gets no target.
    Rows (pixels; g = the stride-8 grid coordinate):
      * g % 1 exactly 0.5 and the next float below, in x and in y;
      * g exactly 1.0 and the next float above; W - g (gxi) and H - g (gyi) exactly 1.0;
      * centres at exactly W and H and at -8 (gi / gj clamped from W / H and from -1, tbox keeps the unclamped cell);
      * l / anchor exactly 4.0 and fp32(3.44) against the 16 x 30 px anchor, and anchor / l exactly 4.0;
      * six targets in one cell, tiny to large, so some rows' CIoU is negative and tobj's clamp(0) matters;
      * angles -90 and 89 degrees (the CSL wrap) among the random ones."""
    rng = np.random.default_rng(seed)
    rows = []   # (cx, cy, l, s)

    def add(cx, cy, l=12.0, s=10.0):
        rows.append((cx, cy, l, s))

    for f in (10.5, _f32_below(10.5)):
        add(8 * f, 8 * 6.25)
        add(8 * 7.25, 8 * f)
    for f in (1.0, _f32_above(1.0)):
        add(8 * f, 8 * 9.25)
        add(8 * 9.25, 8 * f)
    add(W - 8.0, 8 * 5.25)
    add(8 * 5.25, H - 8.0)
    add(float(W), 8 * 3.25, 40.0, 30.0)
    add(8 * 3.25, float(H), 40.0, 30.0)
    add(-8.0, 8 * 4.75, 40.0, 30.0)
    add(8 * 4.75, -8.0, 40.0, 30.0)
    add(float(W), float(H), 24.0, 24.0)
    add(-8.0, -8.0, 24.0, 24.0)
    for r in (4.0, float(np.float32(3.44))):
        add(8 * 12.25, 8 * 2.75, float(np.float32(16 * np.float32(r))), 30.0)
    add(8 * 14.25, 8 * 2.75, 4.0, 30.0)
    for l, s in ((3.0, 4.0), (30.0, 6.0), (10.0, 13.0), (60.0, 50.0), (3.0, 40.0), (24.0, 4.0)):
        add(8 * 6.25 + rng.uniform(0, 6), 8 * 10.75 + rng.uniform(0, 1.5), l, s)
    nt = len(rows) + 12
    t = np.zeros((nt, 187), np.float32)
    t[: len(rows), 2:6] = rows
    t[len(rows):, 2] = rng.uniform(0, W, nt - len(rows))
    t[len(rows):, 3] = rng.uniform(0, H, nt - len(rows))
    t[len(rows):, 4] = np.exp(rng.uniform(np.log(8), np.log(200), nt - len(rows)))
    t[len(rows):, 5] = t[len(rows):, 4] * rng.uniform(0.15, 1.0, nt - len(rows))
    t[:, 0] = rng.integers(0, max(B - 1, 1), nt)
    t[:, 1] = rng.integers(0, nc, nt)
    k = rng.integers(0, 180, nt)
    k[:4] = (0, 179, 0, 179)
    theta = (k - 90) / 180 * PI
    t[:, 6] = theta
    for i in range(nt):
        t[i, 7:] = gaussian_label(theta[i] * 180 / PI + 90)
    return t


def tie_targets(B, H, W, nc=15, seed=0):
    """[nt, 187] targets whose CIoU ties with the predicted box of zero box logits (centre = cell + 0.5, size = the anchor) at
    the 10 x 13 px stride-8 anchor: equal x edges (or y edges) with the other axis unequal, and an overlap width of exactly 0
    from either side (the target starts where the predicted box ends), reached through the neighbour-cell rows.  (A zero
    overlap height needs a target under 1/4 of the anchor's height, which the anchor test rejects.)  W >= 264, H >= 200."""
    rows = [(8 * 20.5, 8 * 8.25, 10.0, 20.0),     # x1 and x2 equal, y unequal
            (8 * 9.25, 8 * 24.5, 24.0, 13.0),     # y1 and y2 equal
            (8 * 31.375, 8 * 12.75, 4.0, 13.0),   # target x1 = predicted x2 in the cell to the left (k = 1 row)
            (8 * 14.625, 8 * 5.75, 4.0, 13.0)]    # target x2 = predicted x1 in the cell to the right (k = 3 row)
    rng = np.random.default_rng(seed)
    t = np.zeros((len(rows), 187), np.float32)
    t[:, 2:6] = rows
    t[:, 0] = rng.integers(0, B, len(rows))
    t[:, 1] = rng.integers(0, nc, len(rows))
    theta = (rng.integers(0, 180, len(rows)) - 90) / 180 * PI
    t[:, 6] = theta
    for i in range(len(rows)):
        t[i, 7:] = gaussian_label(theta[i] * 180 / PI + 90)
    return t


def synth_preds(B, imgsz, no=200, seed=0, na=3, scale=1.5, W=None):
    g = torch.Generator().manual_seed(seed)
    W = imgsz if W is None else W
    return [torch.randn(B, na, imgsz // s, W // s, no, generator=g) * scale for s in (8, 16, 32)]


CLOSEAUG_HYP = dict(box=0.0539, cls=0.299, cls_pw=0.825, obj=0.632, obj_pw=1.0, theta=0.299, theta_pw=0.825, anchor_t=3.44,
                    fl_gamma=0.0, label_smoothing=0.0)   # data/hyps/obb/hyp.finetune_dota_CloseAug.yaml


def _saturate(p, seed):
    """A third of every logit but w / h (channels 2, 3) set to +-20, +-40 or +-90.  A saturated w / h logit makes a predicted box
    of width 2^-56 (x = -20) down to exactly 0 in fp32 (x < -88.7), whose CIoU gradient fp32 cannot follow."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for x in p:
        v = torch.tensor([-90.0, -40.0, -20.0, 20.0, 40.0, 90.0])[torch.randint(0, 6, x.shape, generator=g)]
        sat = torch.rand(x.shape, generator=g) < 1 / 3
        sat[..., 2:4] = False
        out.append(torch.where(sat, v, x))
    return out


def compact_layouts(tg):
    """The 187-, 8- and 7-column forms of [nt, 187] targets (8: the rotation index from the fp32 theta, as the caller would)."""
    from yolov5_obb_b200.loss import compact_csl_index
    t8 = torch.cat([tg[:, :7], torch.from_numpy(compact_csl_index(tg[:, 6].double().numpy())).view(-1, 1)], 1)
    return {187: tg, 8: t8, 7: tg[:, :7].contiguous()}


def exact_cases():
    """name -> (fp32 predictions, targets, hyp, nc): the loss inputs checked element by element against fp64.  Built lazily."""
    from oracle.loss_ref import DEFAULT_HYP, scaled_hyp

    def hyp(base, nc, imgsz, **kw):
        return dict(scaled_hyp(dict(DEFAULT_HYP, **base), 3, nc, imgsz), **kw)

    B, H, W = 3, 256, 320
    bt = torch.from_numpy(boundary_targets(B, H, W, seed=1))
    lay = compact_layouts(bt)
    small = synth_targets(2, 40, 256, seed=3)
    small[:, 4] = np.float32(np.random.default_rng(3).uniform(4, 10, 40))
    small[:, 5] = small[:, 4] * np.float32(0.8)
    tie_p = synth_preds(2, H, seed=6, W=W)
    for x in tie_p:
        x[..., :4] = 0.0
    return {
        "boundary-187": lambda: (synth_preds(B, H, seed=1, W=W), lay[187], hyp({}, 15, W), 15),
        "boundary-8": lambda: (synth_preds(B, H, seed=1, W=W), lay[8], hyp({}, 15, W), 15),
        "boundary-7": lambda: (synth_preds(B, H, seed=1, W=W), lay[7], hyp({}, 15, W), 15),
        "boundary-closeaug": lambda: (synth_preds(B, H, seed=2, W=W), bt, hyp(CLOSEAUG_HYP, 15, W), 15),
        "boundary-smooth": lambda: (synth_preds(B, H, seed=3, W=W), bt, hyp({}, 15, W, label_smoothing=0.1), 15),
        "boundary-nc7": lambda: (synth_preds(B, H, no=192, seed=4, W=W),
                                 torch.from_numpy(boundary_targets(B, H, W, nc=7, seed=2)), hyp({}, 7, W), 7),
        "saturated": lambda: (_saturate(synth_preds(B, H, seed=5, W=W), 5), bt, hyp(CLOSEAUG_HYP, 15, W), 15),
        "ties": lambda: (tie_p, torch.from_numpy(tie_targets(2, H, W, seed=4)), hyp({}, 15, W), 15),
        "p5-no-rows": lambda: (synth_preds(2, 256, seed=7), torch.from_numpy(small), hyp({}, 15, 256), 15),
        "nt1": lambda: (synth_preds(2, 256, seed=8), torch.from_numpy(synth_targets(2, 1, 256, seed=8)), hyp({}, 15, 256), 15),
    }
