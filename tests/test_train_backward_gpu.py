"""GPU parity of the training backward pass (BN/SiLU backward, wgmma dgrad + wgrad, pool / upsample / Detect
backward) against autograd over the fp32 oracle (oracle/model_ref), which is what the reference runs under
train.py:333.

A freshly initialised network with batch-statistic BatchNorm is chaotic: rounding activations to bf16 where the device
stores them moves the fp32 oracle's OWN parameter gradients by ~40 % (test_noise_floor_documented measures it), so
an end-to-end gradient comparison cannot separate a defect from storage noise.  The parity test therefore is TEACHER
FORCED, one module deep: every module (Conv / C3 / SPPF / Detect) is re-evaluated in fp32 on the inputs the device
produced, its output receives the gradient the device held for that output, and autograd's parameter gradients and
input gradients are compared with the device's.  Every parameter gradient and every gradient buffer of the plan is
covered.  Tolerance (bf16 storage inside a module, up to 8 convolutions deep): relative L2 error < 6e-2 per tensor,
median < 2e-2."""
import copy

import pytest
import torch
import torch.nn.functional as F

from oracle import model_ref
from tests.modelgen import build_mirror
from yolov5_obb_b200.layout import sources
from yolov5_obb_b200.train_engine import _PoolLayer
import yolov5_obb_b200.yolo as Y

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _nchw(s):
    return s.buf[..., s.c_off:s.c_off + s.C].float().permute(0, 3, 1, 2).contiguous().cpu()


def _teacher_forced(md, ref_m, eng, x, G):
    """-> (expected parameter grads by name, {layer index: expected gradient of that layer's output})."""
    mods = list(ref_m.model)
    real = {i for i, m in enumerate(mods) if isinstance(m, (Y.Conv, Y.C3, Y.SPPF))}
    leaves = {i: _nchw(eng.out_slices[i]).requires_grad_(True) for i in real}
    plan = eng._bwd

    def gout(i):
        s = eng.out_slices[i]
        gb = plan.gbuf[s.buf.data_ptr()]
        return gb[..., s.c_off:s.c_off + s.C].float().permute(0, 3, 1, 2).contiguous().cpu()

    def resolve(j):
        m = mods[j]
        if j in real:
            return leaves[j]
        if isinstance(m, Y.Concat):
            return torch.cat([resolve(s) for s in sources(m)], 1)
        if isinstance(m, Y.Upsample):
            return F.interpolate(resolve(sources(m)[0]), scale_factor=2, mode="nearest")
        raise AssertionError(type(m))

    ref_m.zero_grad()
    total = 0.0
    extra = {}
    with torch.enable_grad():
        for i, m in enumerate(mods):
            if i in real:
                xin = x.bfloat16().float() if i == 0 else resolve(sources(m)[0])
                if isinstance(m, Y.SPPF):
                    # two teacher-forced pieces: cv1 | max-pools + cv2 on the device's own cv1 output (the arg-max
                    # of a max-pool is decided by the STORED bf16 values; recomputing them in fp32 would move maxima)
                    cat4 = [l for l in eng.layers if isinstance(l, _PoolLayer)][0].cat4
                    c_ = m.cv1.conv.out_channels
                    y1 = cat4[..., :c_].float().permute(0, 3, 1, 2).contiguous().cpu().requires_grad_(True)
                    g_y1 = plan.gbuf[cat4.data_ptr()][..., :c_].float().permute(0, 3, 1, 2).contiguous().cpu()
                    total = total + (model_ref.conv_fwd(m.cv1, xin, True) * g_y1).sum()
                    p1 = F.max_pool2d(y1, 5, 1, 2)
                    p2 = F.max_pool2d(p1, 5, 1, 2)
                    out = model_ref.conv_fwd(m.cv2, torch.cat([y1, p1, p2, F.max_pool2d(p2, 5, 1, 2)], 1), True)
                    total = total + (out * gout(i)).sum()
                    extra[i] = (y1, g_y1)
                    continue
                fn = {Y.Conv: model_ref.conv_fwd, Y.C3: model_ref.c3_fwd}[type(m)]
                total = total + (fn(m, xin, True) * gout(i)).sum()
            elif isinstance(m, Y.Detect):
                outs = model_ref.detect_fwd(m, [resolve(f) for f in m.f], True)
                total = total + sum((o * g).sum() for o, g in zip(outs, G))
        total.backward()
    pg = {n: p.grad.clone() for n, p in ref_m.named_parameters()}
    # layer 23 etc. feed only Detect; the stem has no input gradient
    inner = {i: (leaf.grad, have) for i, (leaf, have) in extra.items()}   # SPPF: gradient of cv1's output
    return pg, {i: leaves[i].grad for i in real if leaves[i].grad is not None}, gout, inner


@pytest.mark.parametrize("size,B,H,W", [("n", 2, 128, 160), ("s", 2, 256, 256), ("m", 1, 64, 96)])
def test_backward_teacher_forced_parity(size, B, H, W):
    m = build_mirror(size, nc=15, seed=3).train()
    ref_m = copy.deepcopy(m)
    g = torch.Generator().manual_seed(11)
    x = torch.rand(B, 3, H, W, generator=g)
    md = m.to(DEV)
    outs = md(x.to(DEV))
    G = [torch.randn(o.shape, generator=g) * 0.05 for o in outs]
    sum((o * gg.to(DEV)).sum() for o, gg in zip(outs, G)).backward()
    torch.cuda.synchronize()
    eng = [e for k, e in md._engines.items() if k[0] == "train"][0]
    pg, gl, gout, inner = _teacher_forced(md, ref_m, eng, x, G)

    rels, bad = [], []
    for n, p in md.named_parameters():
        assert p.grad is not None, n
        a, b = p.grad.float().cpu(), pg[n]
        rel = (a - b).norm().item() / max(b.norm().item(), 1e-12)
        rels.append(rel)
        if rel >= 6e-2:
            bad.append((n, rel))
    rels.sort()
    print(f"{size}: {len(rels)} parameter tensors: median rel {rels[len(rels) // 2]:.3g}, max {rels[-1]:.3g}")
    assert not bad, bad[:10]
    assert rels[len(rels) // 2] < 2e-2
    grels = []
    for i, ref in sorted(gl.items()):
        a = gout(i)
        rel = (a - ref).norm().item() / max(ref.norm().item(), 1e-12)
        grels.append((rel, i))
    print("gradient buffers:", " ".join(f"{i}:{r:.3f}" for r, i in grels))
    assert max(r for r, _ in grels) < 6e-2, grels
    for i, (want, have) in inner.items():
        rel = (have - want).norm().item() / max(want.norm().item(), 1e-12)
        print(f"SPPF {i}: gradient of cv1's output through the three max-pools: rel {rel:.3g}")
        assert rel < 3e-2


def test_noise_floor_documented():
    """The fp32 oracle against ITSELF with bf16 storage emulated: the end-to-end parameter gradients move by tens of
    percent — the reason the parity test above is teacher forced.  (CPU only; kept next to the test it justifies.)"""
    m = build_mirror("n", nc=15, seed=3).train()
    g = torch.Generator().manual_seed(11)
    x = torch.rand(2, 3, 128, 160, generator=g)

    def grads(emul):
        mm = copy.deepcopy(m)
        with torch.enable_grad():
            outs = model_ref.forward_with_grad(mm, x, training=True, emulate_bf16=emul)
            sum(torch.sigmoid(o).mean() for o in outs).backward()
        return {n: p.grad for n, p in mm.named_parameters()}

    a, b = grads(False), grads(True)
    rels = sorted(((a[n] - b[n]).norm() / a[n].norm().clamp_min(1e-20)).item() for n in a)
    print("median relative move of the oracle's own gradients under bf16 storage:", rels[len(rels) // 2])
    assert rels[len(rels) // 2] > 0.1


def test_grads_accumulate_and_second_step_runs():
    """A second backward accumulates into .grad (autograd semantics) and the plan is reusable after a weight update."""
    m = build_mirror("n", nc=15, seed=4).train().to(DEV)
    g = torch.Generator().manual_seed(5)
    x = torch.rand(2, 3, 64, 64, generator=g).to(DEV)
    outs = m(x)
    G = [torch.randn(o.shape, generator=g).to(DEV) * 0.05 for o in outs]
    sum((o * gg).sum() for o, gg in zip(outs, G)).backward()
    g1 = {n: p.grad.clone() for n, p in m.named_parameters()}
    outs = m(x)
    sum((o * gg).sum() for o, gg in zip(outs, G)).backward()
    torch.cuda.synchronize()
    for n, p in m.named_parameters():  # split-K / reduction atomics reorder fp32 sums: equal up to rounding noise
        rel = (p.grad - 2 * g1[n]).norm().item() / max(g1[n].norm().item(), 1e-12)
        assert rel < 2e-2, (n, rel)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(p.grad, alpha=-1e-3)
    m.zero_grad()
    outs2 = m(x)
    sum((o * gg).sum() for o, gg in zip(outs2, G)).backward()
    torch.cuda.synchronize()
    assert all(torch.isfinite(p.grad).all() for p in m.parameters())
