"""fp64 reference and per-element error bounds for the training loss (csrc/loss.cu), forward and backward.

The reference is oracle/loss_ref.compute_loss called on the CPU with fp64 predictions and the fp32 targets: build_targets makes
every matching decision in fp32, as the reference does; CIoU, the BCE terms and autograd run in fp64; tobj follows the CPU rule
that the last write wins.  Each bound is a stated multiple of u = 2^-24 times a magnitude computed in fp64 from the same inputs:

  * BCE gradient (cls, theta, obj): g = scale (s (1 + (pw - 1) t) - pw t), s = sigmoid(x), scale = grad_loss B gain / (n nc)
    (theta: / (n 180), obj: balance / cells).  The sigmoid (expf, an add, a divide), the weight, the product and difference, and
    scale's own five roundings are about 16 roundings; doubled: K_BCE u |scale| (s (1 + (pw - 1) t) + pw t), K_BCE = 32, plus
    |scale| (2 + (pw - 1) t) 2^-48: the fp64 reference's own error, a few 2^-53 of the O(1) terms torch's BCE backward adds
    (at x = -90, t = 0 it returns about -1e-34 |scale| for an exact 8e-40 |scale|); it also covers an fp32 sigmoid
    that is 0 below x = -88.7.  And 2^-146 per row (8 subnormal ulps) for gradients whose last roundings fall below 2^-126.
    Rows that share a cell add into it with atomics: (K_BCE + count - 1) u times the sum of the rows' magnitudes.
  * The saturated case leaves the w / h logits unsaturated (tests/lossgen._saturate): below about -20 the predicted box is
    narrower than 2^-56 anchors, and fp32 cannot hold its CIoU gradient to these bounds.
  * CIoU value: every box edge is formed with an absolute error of a few u M (M the largest |edge|); the overlap width, the
    enclosing width, the centre distance and w / h each carry it, divided by a width of at least S (the smallest side of the two
    boxes), plus about 20 roundings of terms bounded by 1: K_CIOU u (1 + M / S), capped at 1 (tobj lies in [0, 1]).
  * obj gradient: the BCE bound plus |scale| |s (pw - 1) - pw| times the CIoU bound of the cell's winning row (t's error).
  * box gradient (channels 0-3): the CIoU chain cancels, so no per-element relative bound exists.  Each row adds C_BOX = 2^-12
    times its largest fp64 box gradient (about 64 roundings along the forward-mode chain, times a cancellation of at most 2^6
    between the IoU, distance and aspect terms), plus K_SIG u J_i |dL/ds_i|: the sigmoid derivative s (1 - s) is formed from an
    fp32 s, whose error is absolute once s nears 1 (J = 2 for x, y; 8 anchor for w, h is the derivative's scale).
  * items: rows are fp32 sums (a lane's terms, then the 5-level warp tree: gamma(ceil(nc / 32) + 5)) summed in double; obj
    partials are 256-wide fp32 trees (gamma(8)); one fp32 rounding for each hyp / balance gain and for the final cast.
  * zeros: every element no term of the loss reaches (outside channel 4 of the cells no row lands in) must be exactly 0.  An
    element a term reaches may still be 0 in fp64 (s rounds to 1 at x = 40); the bound holds it.
"""
import contextlib
import math

import numpy as np
import torch

from oracle import loss_ref
from tests.losscases import ANCHORS_GRID, STRIDES

U = 2.0 ** -24
K_BCE = 32
K_CIOU = 64
C_BOX = 2.0 ** -12
K_SIG = 8
SUBNORMAL = 2.0 ** -146   # 8 ulps of fp32's subnormal range: a gradient element whose last roundings fall below 2^-126
REF_ABS = 2.0 ** -48     # the fp64 reference's own absolute error in a BCE gradient: a few 2^-53 of its O(1) terms
BALANCE = (4.0, 1.0, 0.4)


def gamma(d: int) -> float:
    return d * U / (1.0 - d * U)


def expand_csl(tg: torch.Tensor, sigma: float = 2.0) -> torch.Tensor:
    """[nt, 187 | 8 | 7] -> [nt, 187]: the CSL row the kernel reads (187) or rebuilds from the rotation index (8: column 7;
    7: int(90 - angle) from the fp32 theta, angle = theta * 180 / 3.141592 + 90 in fp64)."""
    tg = tg.float()
    if tg.shape[1] >= 187:
        return tg
    y = torch.from_numpy(np.exp(-((np.arange(180) - 90.0) ** 2) / (2 * sigma * sigma)).astype(np.float32))
    if tg.shape[1] == 8:
        idx = tg[:, 7].double().trunc().long()
    else:
        idx = (90.0 - (tg[:, 6].double() * 180.0 / 3.141592 + 90.0)).trunc().long()
    j = (torch.arange(180)[None] + idx[:, None]) % 180
    return torch.cat([tg[:, :7], y[j]], 1)


@contextlib.contextmanager
def serial():
    """One CPU thread: ATen's CPU index_put_ without accumulate splits the indices across threads, and the last write on a
    duplicated cell (tobj's rule) is only the last row when one thread writes them all."""
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        yield
    finally:
        torch.set_num_threads(n)


def reference(p, tg, hyp, nc, anchors=ANCHORS_GRID, strides=STRIDES):
    """fp64 (loss [1], items [4], dense gradients for grad_loss = 1) of the predictions p (list of [B, na, H, W, no])."""
    p64 = [x.detach().cpu().double().requires_grad_(True) for x in p]
    with serial():
        loss, items = loss_ref.compute_loss(p64, expand_csl(tg.cpu()), anchors, strides, hyp, nc)
    loss.backward()
    return loss.detach(), items, [x.grad for x in p64]


def _bce_parts(x, t, pw):
    """fp64 (gradient magnitude s lw + pw t, d grad / dt, value magnitude, d value / dt) of BCEWithLogits."""
    s = torch.sigmoid(x)
    lw = 1 + (pw - 1) * t
    sp = torch.log1p(torch.exp(-x.abs())) + (-x).clamp(min=0)
    return (s * lw + pw * t + (1 + lw) * REF_ABS / (K_BCE * U), (s * (pw - 1) - pw).abs(), ((1 - t) * x).abs() + lw * sp,
            (-x + (pw - 1) * sp).abs())


def _ciou_rows(ps, tbox, anch):
    """Per row: fp64 CIoU, dCIoU/dlogit [n, 4], dCIoU/dsigmoid [n, 4] and the CIoU value bound."""
    x = ps[:, :4].detach().clone().requires_grad_(True)
    s = x.sigmoid()
    s.retain_grad()
    pxy = s[:, :2] * 2 - 0.5
    pwh = (s[:, 2:4] * 2) ** 2 * anch.double()
    pbox = torch.cat((pxy, pwh), 1)
    tb = tbox.double()
    ciou = loss_ref.bbox_ciou(pbox.T, tb)
    ciou.sum().backward()
    edges = torch.cat([pbox[:, :2].abs() + pbox[:, 2:] / 2, tb[:, :2].abs() + tb[:, 2:] / 2], 1)
    M = edges.max(1).values
    S = torch.cat([pbox[:, 2:], tb[:, 2:]], 1).min(1).values
    dc = (K_CIOU * U * (1 + M / S)).nan_to_num(1.0).clamp(max=1.0)
    return ciou.detach(), x.grad, s.grad, dc.detach()


def bounds(p, tg, hyp, nc, anchors=ANCHORS_GRID, strides=STRIDES):
    """Per-element bounds for grad_loss = 1 (they scale with it) and the item / loss bounds.

    Returns dict(obj=[per level [B, na, H, W] bound of channel 4], cells=[per level flat indices of the cells rows land in],
    rows=[per level [len(cells), no] bound of every other channel of those cells], items=[4], loss=float, nrows=[per level]).
    """
    p64 = [x.detach().cpu().double() for x in p]
    tg187 = expand_csl(tg.cpu())
    B, na = p64[0].shape[:2]
    no = p64[0].shape[-1]
    ci = 5 + nc
    tcls, tbox, indices, anch, tcsl = loss_ref.build_targets(p64, tg187, anchors, strides, hyp["anchor_t"], na)
    cp, cn = 1.0 - 0.5 * hyp.get("label_smoothing", 0.0), 0.5 * hyp.get("label_smoothing", 0.0)
    pws = {k: float(hyp.get(k, 1.0)) for k in ("cls_pw", "obj_pw", "theta_pw")}
    out = dict(obj=[], cells=[], rows=[], nrows=[])
    e_items = [0.0, 0.0, 0.0, 0.0]
    for i, pi in enumerate(p64):
        _, _, H, W, _ = pi.shape
        ncell = B * na * H * W
        b, a, gj, gi = indices[i]
        n = b.shape[0]
        out["nrows"].append(n)
        flat = ((b * na + a) * H + gj) * W + gi
        tobj = torch.zeros(B, na, H, W, dtype=torch.float64)
        dt = torch.zeros(B, na, H, W, dtype=torch.float64)
        cells = torch.unique(flat)
        rb = torch.zeros(cells.numel(), no, dtype=torch.float64)
        if n:
            pos = torch.searchsorted(cells, flat)
            count = torch.bincount(pos, minlength=cells.numel()).double()
            ps = pi[b, a, gj, gi]
            ciou, gx, gs, dc = _ciou_rows(ps, tbox[i], anch[i])
            with serial():                         # the same sequential writes as loss_ref: the same winner per cell
                tobj[b, a, gj, gi] = ciou.clamp(0)
                dt[b, a, gj, gi] = dc
            # box channels
            sb = B * hyp["box"] / n
            g_row = (sb * gx).abs()
            J = torch.stack([torch.full_like(anch[i][:, 0], 2.0), torch.full_like(anch[i][:, 0], 2.0),
                             8 * anch[i][:, 0], 8 * anch[i][:, 1]], 1).double()
            per = C_BOX * g_row.max(1, keepdim=True).values + K_SIG * U * J * (sb * gs).abs()
            rb[:, :4].index_add_(0, pos, per)
            box_sum = torch.zeros(cells.numel(), 4, dtype=torch.float64).index_add_(0, pos, g_row)
            rb[:, :4] += (count - 1)[:, None] * U * box_sum
            e_items[0] += float(((dc + U * (1 - ciou).abs()).sum()) / n)
            # class and theta channels
            mag = torch.zeros(cells.numel(), no, dtype=torch.float64)
            if nc > 1:
                t = torch.full((n, nc), cn, dtype=torch.float64)
                t[range(n), tcls[i]] = cp
                gm, _, vm, _ = _bce_parts(ps[:, 5:ci], t, pws["cls_pw"])
                mag[:, 5:ci].index_add_(0, pos, B * hyp["cls"] / (n * nc) * gm)
                e_items[2] += float(((K_BCE * U + gamma(-(-nc // 32) + 5)) * vm.sum(1)).sum() / (n * nc))
            gm, _, vm, _ = _bce_parts(ps[:, ci:], tcsl[i].double(), pws["theta_pw"])
            mag[:, ci:].index_add_(0, pos, B * hyp["theta"] / (n * 180) * gm)
            e_items[3] += float(((K_BCE * U + gamma(6 + 5)) * vm.sum(1)).sum() / (n * 180))
            rb[:, 5:] += (K_BCE + count - 1)[:, None] * U * mag[:, 5:] + count[:, None] * SUBNORMAL
        # obj channel, every cell
        so = B * hyp["obj"] * BALANCE[i] / ncell
        gm, dgt, vm, dvt = _bce_parts(pi[..., 4], tobj, pws["obj_pw"])
        out["obj"].append(K_BCE * U * so * gm + so * dgt * dt + SUBNORMAL)
        e_lvl = (K_BCE * U * vm + dvt * dt).sum() + (gamma(8) + ncell * 2.0 ** -53) * vm.sum()
        e_items[1] += float(e_lvl) / ncell * BALANCE[i]
        out["cells"].append(cells)
        out["rows"].append(rb)
    gains = (hyp["box"], hyp["obj"], hyp["cls"], hyp["theta"])
    with serial():
        _, items64 = loss_ref.compute_loss(p64, tg187, anchors, strides, hyp, nc)
    items64 = items64.tolist()
    out["items"] = [e * g + 4 * U * abs(v) for e, g, v in zip(e_items, gains, items64)]
    out["loss"] = B * (sum(out["items"]) + 4 * U * sum(abs(v) for v in items64))
    return out


def check(grads, loss, items, ref, bnd, gl=1.0):
    """Compare one run (dense grads for grad_loss = gl [per level, same shape as p], loss [1], items [4]; any device) with the
    fp64 reference (reference()'s output) under `bnd` (bounds()'s output).  Returns the worst error / bound of each element
    class; raises AssertionError naming the first class past its bound, or a non-zero element that no term reaches."""
    loss64, items64, g64s = ref
    worst = {}

    def note(k, err, bound):
        if err.numel():
            ratio = torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, math.inf, 0.0))
            worst[k] = max(worst.get(k, 0.0), float(ratio.max()))
        assert worst.get(k, 0.0) <= 1.0, f"{k}: error / bound = {worst[k]:.3g}"

    it = items.detach().double().cpu()
    note("items", (it - items64).abs(), torch.tensor(bnd["items"], dtype=torch.float64))
    note("loss", (loss.detach().double().cpu() - loss64).abs(), torch.tensor([bnd["loss"]]))
    for i, (g, g64) in enumerate(zip(grads, g64s)):
        dev = g.device
        g64d = g64.to(dev) * gl
        gd = g.detach().double()
        no = g.shape[-1]
        cells = bnd["cells"][i].to(dev)
        reached = torch.zeros(gd.numel() // no, no, dtype=torch.bool, device=dev)
        reached[:, 4] = True
        reached[cells] = True
        reached = reached.view(gd.shape)
        assert bool((g64d[~reached] == 0).all())
        bad = int((gd[~reached] != 0).sum())
        assert bad == 0, f"level {i}: {bad} elements non-zero that no term of the loss reaches"
        err = (gd - g64d).abs()
        note("obj", err[..., 4], bnd["obj"][i].to(dev) * gl)
        er = err.reshape(-1, no)[cells]
        rb = bnd["rows"][i].to(dev) * gl
        nc = no - 185
        note("box", er[:, :4], rb[:, :4])
        if nc > 1:
            note("cls", er[:, 5:5 + nc], rb[:, 5:5 + nc])
        note("theta", er[:, 5 + nc:], rb[:, 5 + nc:])
    return worst
