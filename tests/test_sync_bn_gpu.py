"""SyncBatchNorm in the training plans (train.py --sync-bn, torch.nn.SyncBatchNorm): the split BatchNorm entry points of
csrc/bn_train.cu, the per-layer collectives of TrainEngine / BackwardPlan and TrainStep(sync_bn=True).

Multi-rank cases run as two spawned processes sharing GPU 0 over gloo on 127.0.0.1 (the plans then run eagerly, with the
collective between launches); the graph-capture case runs one NCCL rank.  Every case has a timeout and joins (or kills)
every process it started.

  1. kernels: world-1 records give the plain entry points' results bit for bit; two "ranks" of unequal pixel counts, their
     records added in fp64, match fp64 BatchNorm over the union (tests/bnref.py bounds);
  2. two identical ranks: activations, Detect logits, loss and the flat gradient before its all-reduce equal a
     single-process plain step bit for bit, running_var follows the 2n count (SGD, --freeze 10, Adam, accumulate 2);
  3. two ranks with different statistics against the fp32 oracle whose batch norm is torch's SyncBatchNorm function over
     the same group, within the bf16-emulated oracle's own drift; the per-rank oracle lies outside that tolerance;
  4. --multi-scale with different sizes per rank: every layer's statistics match fp64 over the union of both ranks' maps,
     and the ranks' running statistics are bit-equal;
  5. a one-rank NCCL group forced through the sync plans: eager, captured and replayed steps equal the plain plans;
  6. TrainStep(sync_bn=True) without a process group or at world size 1 is TrainStep(sync_bn=False)."""
import copy
import os
import socket
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import bnref
from tests.bnref import U, gamma, stat_chain, ulp32
from tests.lossgen import synth_targets
from tests.modelgen import build_mirror
from tests.tilegen import synth_tiles

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS, MOM = 1e-3, 0.03
S = 128          # image size of the multi-rank cases (yolov5n)
TIMEOUT = 600


# ====================================================================================================== process harness
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _entry(fn, rank, ws, port, backend, q, args):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(ws))
    try:
        dev = torch.device("cuda", rank if backend == "nccl" else 0)
        torch.cuda.set_device(dev)
        kw = dict(device_id=dev) if backend == "nccl" else {}
        dist.init_process_group(backend, rank=rank, world_size=ws, **kw)
        try:
            q.put((rank, "ok", fn(rank, ws, *args)))
        finally:
            dist.destroy_process_group()
    except BaseException:
        q.put((rank, "error", traceback.format_exc()))


def spawn(fn, ws=2, *args, backend="gloo"):
    """fn(rank, ws, *args) in `ws` spawned ranks -> its return values (picklable, host data) in rank order."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_entry, args=(fn, r, ws, port, backend, q, args)) for r in range(ws)]
    for p in procs:
        p.start()
    res = []
    try:
        for _ in range(ws):
            res.append(q.get(timeout=TIMEOUT))
    finally:
        for p in procs:
            p.join(60)
            if p.is_alive():
                p.kill()
                p.join()
    bad = [r for r in res if r[1] != "ok"]
    assert not bad, "\n".join(f"rank {r}:\n{msg}" for r, _, msg in bad)
    assert all(p.exitcode == 0 for p in procs)
    return [out for _, _, out in sorted(res, key=lambda r: r[0])]


def host(t):
    """A device tensor as a numpy array that keeps its bits (bf16 as int16)."""
    t = t.detach()
    if t.dtype == torch.bfloat16:
        t = t.view(torch.int16)
    return t.cpu().numpy().copy()


def batch(B=2, seed=3, gain=1.0):
    imgs = synth_tiles(B, S, seed=seed)
    if gain != 1.0:
        imgs = (imgs.float() * gain).round().clamp(0, 255).to(torch.uint8)
    return imgs, torch.from_numpy(synth_targets(B, 20, S, nc=15, seed=seed))


WGRAD_RTOL = 1e-5   # run-to-run spread of a weight gradient: wgrad_kernel adds its split-K slices with fp32 atomics


def grad_parts(flat, m):
    """The flat gradient split per parameter: {name: array}.  Every entry is produced by deterministic kernels (BatchNorm
    dgamma / dbeta, the Detect biases' sums, every data gradient on the way) except the conv weights' (wgrad_kernel's fp32
    atomics), which equal another run's only to rounding."""
    from yolov5_obb_b200.train_engine import flat_layout
    names = [n for n, _ in m.named_parameters()]
    offs, _ = flat_layout(list(m.parameters()))
    return {n: flat[o:o + p.numel()] for n, o, p in zip(names, offs, m.parameters())}


def same_grads(a, b, what):
    """Bit-equal gradients of BatchNorm parameters and biases; conv weights within WGRAD_RTOL (relative L2 per tensor)."""
    worst = 0.0
    for n in a:
        if n.endswith("conv.weight") or (n.endswith(".weight") and ".bn." not in n):
            r = float(np.linalg.norm(a[n] - b[n]) / max(np.linalg.norm(a[n]), 1e-30))
            worst = max(worst, r)
            assert r <= WGRAD_RTOL, f"{what}: {n} differs by {r:.2e} relative"
        else:
            assert np.array_equal(a[n], b[n]), f"{what}: {n} differs"
    return worst


def bn_state(m):
    return [torch.cat([b.running_mean, b.running_var]).clone() for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d)]


# =========================================================================================================== 1. kernels
def _lib():
    from yolov5_obb_b200 import _lib as L
    return L.lib()


def _st():
    from yolov5_obb_b200 import _lib as L
    return L.stream_ptr(torch.device(DEV))


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def test_kernels_world_one_bit_exact_and_two_ranks_against_fp64():
    """Every BatchNorm launch of the yolov5s b3 256x320 train plan (the benchmarked yolov5s layers at a small batch), as
    TrainEngine._forward_eager issues it.  World 1: y5obb_bn_stats_sync + y5obb_bn_finalize_sync and
    y5obb_bn_silu_bwd_reduce_sync + y5obb_bn_silu_bwd_apply_sync give y5obb_bn_batch_stats / y5obb_bn_silu_bwd's outputs bit
    for bit.  Two ranks (image 0 and images 1-2: unequal pixel counts), records added in fp64: mean, invstd, scale, shift,
    running statistics and dz against fp64 BatchNorm over all three images."""
    from tests.test_train_plans_pointwise_gpu import _Recorder, _plan, _randomise_bn, gen_z
    m, eng = _plan("s", 3, 256, 320)
    g = torch.Generator(device=DEV).manual_seed(11)
    _randomise_bn(m, g)
    real, rec = eng._L, _Recorder()
    eng._L = rec
    try:
        eng._forward_eager(torch.zeros(3, 3, 256, 320, device=DEV))
    finally:
        eng._L = real
    stats = [a for n, a in rec.calls if n == "y5obb_bn_batch_stats"]
    assert len(stats) == len(eng.conv_layers) > 50
    L, st, sms = _lib(), _st(), _sms()
    scr = eng.scratch
    worst = {}

    def note(k, r):
        worst[k] = max(worst.get(k, 0.0), float(r))
        assert r <= 1.0, f"{k}: error {r:.3f} x its bound"

    def f32(C):
        return torch.full((C,), float("nan"), dtype=torch.float32, device=DEV)

    for i, (lay, sa) in enumerate(zip(eng.conv_layers, stats)):
        z = lay.z
        zp, zs, npix, C = sa[0], sa[1], sa[2], sa[3]
        assert (zp, zs, npix, C) == (z.ptr, z.pix_stride, z.B * z.H * z.W, z.C)
        z.view().copy_(gen_z((z.B, z.H, z.W), C, (0, 3, 10)[i % 3], g))
        bn = lay.mod.bn
        gam, bet = bn.weight.detach(), bn.bias.detach()
        rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
        act = int(lay.act)

        def fwd_plain():
            o = dict(rm=rm0.clone(), rv=rv0.clone(), scale=f32(C), shift=f32(C), mean=f32(C), invstd=f32(C))
            assert L.y5obb_bn_batch_stats(zp, zs, npix, C, gam.data_ptr(), bet.data_ptr(), EPS, MOM, o["rm"].data_ptr(),
                                          o["rv"].data_ptr(), o["scale"].data_ptr(), o["shift"].data_ptr(),
                                          o["mean"].data_ptr(), o["invstd"].data_ptr(), scr.data_ptr(), scr.numel(), st) == 0
            return o

        def rec_fwd(p0, p1):
            r = torch.full((2 * C + 1,), float("nan"), dtype=torch.float64, device=DEV)
            assert L.y5obb_bn_stats_sync(zp + 2 * p0 * zs, zs, p1 - p0, C, r.data_ptr(), scr.data_ptr(), scr.numel(), st) == 0
            return r

        def fin(r):
            o = dict(rm=rm0.clone(), rv=rv0.clone(), scale=f32(C), shift=f32(C), mean=f32(C), invstd=f32(C))
            assert L.y5obb_bn_finalize_sync(r.data_ptr(), C, gam.data_ptr(), bet.data_ptr(), EPS, MOM, o["rm"].data_ptr(),
                                            o["rv"].data_ptr(), o["scale"].data_ptr(), o["shift"].data_ptr(),
                                            o["mean"].data_ptr(), o["invstd"].data_ptr(), st) == 0
            return o

        plain, r1 = fwd_plain(), rec_fwd(0, npix)
        one = fin(r1)
        for k in plain:
            assert torch.equal(plain[k].view(torch.int32), one[k].view(torch.int32)), f"layer {i} {k}: world 1 differs"
        # ---- backward, world 1
        dy = (0.5 * torch.randn((npix, C), device=DEV, generator=g)).bfloat16()
        zt = z.view().reshape(npix, C)

        def bwd_plain():
            s1, s2, dz = f32(C), f32(C), torch.empty((npix, C), dtype=torch.bfloat16, device=DEV)
            dg, db = f32(C), f32(C)
            assert L.y5obb_bn_silu_bwd(zp, zs, dy.data_ptr(), C, npix, C, plain["scale"].data_ptr(),
                                       plain["shift"].data_ptr(), plain["mean"].data_ptr(), plain["invstd"].data_ptr(), act,
                                       s1.data_ptr(), s2.data_ptr(), dz.data_ptr(), C, None, 0, 0, dg.data_ptr(),
                                       db.data_ptr(), 0, scr.data_ptr(), scr.numel(), st) == 0
            return dz, dg, db

        def bwd_reduce(o, p0, p1):
            r = torch.full((2 * C,), float("nan"), dtype=torch.float64, device=DEV)
            dg, db = f32(C), f32(C)
            assert L.y5obb_bn_silu_bwd_reduce_sync(zp + 2 * p0 * zs, zs, dy[p0:].data_ptr(), C, p1 - p0, C,
                                                   o["scale"].data_ptr(), o["shift"].data_ptr(), o["mean"].data_ptr(),
                                                   o["invstd"].data_ptr(), act, r.data_ptr(), dg.data_ptr(), db.data_ptr(), 0,
                                                   scr.data_ptr(), scr.numel(), st) == 0
            return r, dg, db

        def bwd_apply(o, r, rf, p0, p1, dz):
            assert L.y5obb_bn_silu_bwd_apply_sync(zp + 2 * p0 * zs, zs, dy[p0:].data_ptr(), C, p1 - p0, C,
                                                  o["scale"].data_ptr(), o["shift"].data_ptr(), o["mean"].data_ptr(),
                                                  o["invstd"].data_ptr(), act, r.data_ptr(), rf[2 * C:].data_ptr(),
                                                  dz[p0:].data_ptr(), C, None, 0, 0, st) == 0

        dz0, dg0, db0 = bwd_plain()
        rb, dg1, db1 = bwd_reduce(one, 0, npix)
        dz1 = torch.empty_like(dz0)
        bwd_apply(one, rb, r1, 0, npix, dz1)
        torch.cuda.synchronize()
        assert torch.equal(dz0.view(torch.int16), dz1.view(torch.int16)), f"layer {i}: world-1 dz differs"
        assert torch.equal(dg0, dg1) and torch.equal(db0, db1), f"layer {i}: world-1 dgamma / dbeta differ"
        # ---- two ranks: image 0 | images 1-2
        cut = npix // 3
        parts = [(0, cut), (cut, npix)]
        rsum = rec_fwd(*parts[0]) + rec_fwd(*parts[1])
        out = fin(rsum)
        n = npix
        assert rsum[2 * C].item() == n
        d = max(stat_chain(p1 - p0, C, sms) for p0, p1 in parts) + 1
        s, q = rsum[:C], rsum[C:2 * C]
        m64, var64, iv64 = bnref.finalize_ref(s, q, n, EPS)
        assert torch.equal(out["mean"], m64.float()), f"layer {i}: mean != (float)(sum / n)"
        note("invstd (ulp of its own sums)", ((out["invstd"].double() - iv64).abs() / ulp32(iv64)).max().item())
        assert torch.equal(out["scale"], (gam.double() * out["invstd"].double()).float())
        fused = bet.double() - out["mean"].double() * out["scale"].double()
        assert (((out["shift"].double() - fused).abs() <= ulp32(fused)) |
                torch.eq(out["shift"], bet - out["mean"] * out["scale"])).all()
        mom1, momf = float(np.float32(1.0 - MOM)), float(np.float32(MOM))
        unb = var64 * n / (n - 1.0)
        for key, new, old in (("rm", out["mean"].double(), rm0), ("rv", unb, rv0)):
            want = mom1 * old.double() + momf * new
            tol = 4 * U * (mom1 * old.double().abs() + momf * new.abs()) + ulp32(want)
            note("running stats", ((out[key].double() - want).abs() / tol).max().item())
        x = zt.double()
        mt = x.mean(0)
        ivt = 1.0 / torch.sqrt(((x - mt) ** 2).mean(0) + float(np.float32(EPS)))
        note("mean vs fp64", ((out["mean"].double() - mt).abs() / (gamma(d) * x.abs().sum(0) / n + ulp32(mt))).max().item())
        note("invstd quality", ((out["invstd"].double() - ivt).abs() / ivt).max().item() / 2 ** -10)
        # backward over the union
        r0, _, _ = bwd_reduce(out, *parts[0])
        r1b, _, _ = bwd_reduce(out, *parts[1])
        rbs = r0 + r1b
        dz = torch.empty_like(dz0)
        for p0, p1 in parts:
            bwd_apply(out, rbs, rsum, p0, p1, dz)
        torch.cuda.synchronize()
        du, e_du = bnref.du_ref(zt, dy, out["scale"], out["shift"], act)
        s1, s2 = rbs[:C].float(), rbs[C:].float()
        bound_s = gamma(d) * du.abs().sum(0) + e_du.sum(0)
        note("sum du", ((rbs[:C] - du.sum(0)).abs() / (1.001 * bound_s).clamp(min=1e-300)).max().item())
        mm, iv = out["mean"].double(), out["invstd"].double()
        bound_q = gamma(d + 3) * iv * ((du * x).abs().sum(0) + mm.abs() * du.abs().sum(0)) + iv * (e_du * (x - mm).abs()).sum(0)
        note("sum du xhat", ((rbs[C:] - iv * (du * (x - mm)).sum(0)).abs() / (1.001 * bound_q).clamp(min=1e-300)).max().item())
        want, tol = bnref.dz_ref(zt, du, e_du, out["scale"], out["mean"], out["invstd"], s1, s2, n)
        note("dz", ((dz.double() - want).abs() / tol).max().item())
    print("\n[sync-bn kernels] worst error / bound:", {k: f"{v:.3e}" for k, v in worst.items()})


# ============================================================================================== 2. identical ranks
CONFIGS = {"sgd": dict(), "freeze10": dict(freeze=[10]), "adam": dict(adam=True), "accumulate2": dict(batch_size=32)}


def _steps_of(cfg):
    return 2 if cfg.get("batch_size", 64) < 64 else 1   # accumulate 2: the second step is the first optimizer step


def _run_identical(ts, m, imgs, tg, steps, flat_of):
    """`steps` TrainStep.step calls -> per step (loss, flat gradient before any all-reduce, per parameter) and, of the last forward,
    every conv layer's output and the Detect logits; the running statistics after the steps."""
    out = []
    for _ in range(steps):
        loss, _ = ts.step(imgs, tg)
        eng = m._last_train_engine
        out.append(dict(loss=host(loss), flat=grad_parts(flat_of(eng), m)))
    eng = m._last_train_engine
    act = [host(lay.y.view()) for lay in eng.conv_layers]
    det = [host(o) for o in eng.det_out]
    return out, act, det, [host(t) for t in bn_state(m)]


def _identical_worker(rank, ws, cfg):
    from yolov5_obb_b200 import train_step
    m = build_mirror("n", nc=15, seed=1).train().to(DEV)
    ts = train_step.TrainStep(m, imgsz=S, **{"batch_size": 64, **cfg}, sync_bn=True)
    assert m.bn_group is not None
    snap = {}
    orig = dist.all_reduce

    def all_reduce(t, *a, **k):     # the flat gradient as the backward left it, before the data-parallel SUM
        eng = getattr(m, "_last_train_engine", None)
        if eng is not None and eng._bwd is not None and t.data_ptr() == eng._bwd.flat.data_ptr():
            snap["flat"] = host(t)
        return orig(t, *a, **k)

    dist.all_reduce = all_reduce
    try:
        imgs, tg = batch()
        res = _run_identical(ts, m, imgs.to(DEV), tg.to(DEV), _steps_of(cfg),
                             lambda eng: snap.pop("flat", None) if "flat" in snap else host(eng._bwd.flat))
    finally:
        dist.all_reduce = orig
    names = {id(mod): n for n, mod in m.named_modules()}
    recs = [(names[id(lay.mod.bn)], host(lay.rec), host(lay.mod.bn.running_var))
            for lay in m._last_train_engine.conv_layers]
    return res, recs


@pytest.mark.parametrize("name", list(CONFIGS))
def test_identical_ranks_equal_the_single_process_step(name):
    cfg = CONFIGS[name]
    from yolov5_obb_b200.train_step import TrainStep
    m = build_mirror("n", nc=15, seed=1).train().to(DEV)
    rv0 = {n: b.running_var.double().cpu().numpy() for n, b in m.named_modules() if isinstance(b, torch.nn.BatchNorm2d)}
    ts = TrainStep(m, imgsz=S, **{"batch_size": 64, **cfg})
    imgs, tg = batch()
    plain, act, det, rs = _run_identical(ts, m, imgs.to(DEV), tg.to(DEV), _steps_of(cfg), lambda eng: host(eng._bwd.flat))
    for rank, ((sync, act_s, det_s, rs_s), recs) in enumerate(spawn(_identical_worker, 2, cfg)):
        for k, (a, b) in enumerate(zip(plain, sync)):
            assert np.array_equal(a["loss"], b["loss"]), (name, rank, k, a["loss"], b["loss"])
            same_grads(a["flat"], b["flat"], f"{name} rank {rank} step {k}")
        assert all(np.array_equal(a, b) for a, b in zip(act, act_s)), f"{name} rank {rank}: activations differ"
        assert all(np.array_equal(a, b) for a, b in zip(det, det_s)), f"{name} rank {rank}: Detect logits differ"
        for li, (a, b) in enumerate(zip(rs, rs_s)):
            C = a.size // 2
            assert np.array_equal(a[:C], b[:C]), f"{name} rank {rank} BN {li}: running_mean differs"
        if _steps_of(cfg) == 1:    # running_var with the unbiased factor of the 2n pixels of both ranks
            for bn_name, r, rv in recs:
                C = rv.size
                n = r[2 * C]
                var = np.maximum(r[C:2 * C] / n - (r[:C] / n) ** 2, 0)
                want = (1 - MOM) * rv0[bn_name] + MOM * var * n / (n - 1)
                err = np.abs(rv.astype(np.float64) - want)
                assert (err <= 4 * np.spacing(np.abs(want).astype(np.float32))).all(), \
                    f"{name} rank {rank} {bn_name}: running_var does not follow the 2n count"


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="NCCL across ranks needs two GPUs")
def test_identical_ranks_over_nccl_on_two_gpus():
    """Case 2 over NCCL, one rank per GPU: the collectives are captured in the forward and backward graphs."""
    from yolov5_obb_b200.train_step import TrainStep
    m = build_mirror("n", nc=15, seed=1).train().to(DEV)
    ts = TrainStep(m, imgsz=S, batch_size=64)
    imgs, tg = batch()
    plain = [host(ts.step(imgs.to(DEV), tg.to(DEV))[0])]
    for got in spawn(_nccl_identical_worker, 2, backend="nccl"):
        assert np.array_equal(plain[0], got[0])


def _nccl_identical_worker(rank, ws):
    from yolov5_obb_b200.train_step import TrainStep
    dev = torch.device("cuda", rank)
    m = build_mirror("n", nc=15, seed=1).train().to(dev)
    ts = TrainStep(m, imgsz=S, batch_size=64, sync_bn=True)
    imgs, tg = batch()
    out = [host(ts.step(imgs.to(dev), tg.to(dev))[0])]
    for _ in range(3):   # eager, captured, replayed
        ts.step(imgs.to(dev), tg.to(dev))
    return out


# ================================================================================= 3. against the reference semantics
class _SyncF:
    """torch.nn.functional for oracle/model_ref.py with batch_norm replaced by torch's SyncBatchNorm function."""

    def __init__(self, F, group, ws):
        self._F, self._group, self._ws = F, group, ws

    def __getattr__(self, name):
        return getattr(self._F, name)

    def batch_norm(self, x, rm, rv, w, b, training, momentum, eps):
        from torch.nn.modules._functions import SyncBatchNorm
        assert training
        return SyncBatchNorm.apply(x, w, b, rm, rv, eps, momentum, self._group, self._ws)


def _oracle_steps(m0, x, tg, steps, sync, emulate, ws):
    from oracle import model_ref, loss_ref
    from yolov5_obb_b200.train_step import HYP_FINETUNE_DOTA, param_groups
    m = copy.deepcopy(m0).to(DEV).train()
    det = m.model[-1]
    hyp = loss_ref.scaled_hyp({k: HYP_FINETUNE_DOTA.get(k, v) for k, v in loss_ref.DEFAULT_HYP.items()}, det.nl, det.nc, S)
    g0, g1, g2 = param_groups(m)
    opt = torch.optim.SGD(g0, lr=HYP_FINETUNE_DOTA["lr0"], momentum=HYP_FINETUNE_DOTA["momentum"], nesterov=True)
    opt.add_param_group({"params": g1, "weight_decay": HYP_FINETUNE_DOTA["weight_decay"]})
    opt.add_param_group({"params": g2})
    rs0 = torch.cat(bn_state(m))
    F0 = model_ref.F
    out = []
    for _ in range(steps):
        if sync:
            model_ref.F = _SyncF(F0, dist.group.WORLD, ws)
        try:
            with torch.enable_grad():
                pred = model_ref.forward_with_grad(m, x, training=True, emulate_bf16=emulate)
                loss, _ = loss_ref.compute_loss(pred, tg, det.anchors, det.stride, hyp, det.nc)
                loss.backward()
        finally:
            model_ref.F = F0
        for p in m.parameters():
            dist.all_reduce(p.grad, op=dist.ReduceOp.SUM)    # DDP: the SUM over ranks of a loss x WORLD_SIZE
        grad = torch.cat([p.grad.flatten() for p in m.parameters()])
        opt.step()
        opt.zero_grad(set_to_none=True)
        out.append(dict(loss=loss.item(), grad=grad.double(), rs=torch.cat(bn_state(m)).double() - rs0.double()))
    return out


def _semantics_worker(rank, ws, steps):
    from yolov5_obb_b200.train_step import TrainStep
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    m0 = build_mirror("n", nc=15, seed=1).train()
    imgs, tg = batch(gain=1.0 if rank == 0 else 0.3)     # rank 1's images much darker: different batch statistics
    x = imgs.float().to(DEV) / 255
    arms = {k: _oracle_steps(m0, x, tg.to(DEV), steps, sync, emu, ws)
            for k, sync, emu in (("ref", True, False), ("emu", True, True), ("per_rank", False, False))}
    md = copy.deepcopy(m0).to(DEV)
    ts = TrainStep(md, batch_size=64, imgsz=S, sync_bn=True)
    rs0 = torch.cat(bn_state(md))
    dev = []
    for _ in range(steps):
        loss, _ = ts.step(imgs.to(DEV), tg.to(DEV))
        plan = md._last_train_engine._bwd      # its flat buffer was all-reduced in place before the fused SGD step
        grad = torch.cat([plan.pgrad[p].flatten() for p in md.parameters()])
        dev.append(dict(loss=loss.item(), grad=grad.double(), rs=torch.cat(bn_state(md)).double() - rs0.double()))
    arms["device"] = dev
    return {k: [dict(loss=s["loss"], grad=s["grad"].cpu().numpy(), rs=s["rs"].cpu().numpy()) for s in v]
            for k, v in arms.items()}


def test_two_ranks_follow_torch_syncbatchnorm():
    """Loss, summed gradient and the running statistics' update over three SGD steps, the device's sync plans against the
    fp32 oracle with torch's SyncBatchNorm, within 3x the bf16-emulated oracle's own drift (running maximum) + 2 % of the
    loss / 1e-3 relative, the yardstick of test_train_step_gpu.py::test_loss_trajectory_against_the_cpu_oracle.  The
    per-rank (plain BatchNorm) oracle must lie outside that tolerance: the check sees the difference."""
    steps = 3
    res = spawn(_semantics_worker, 2, steps)

    def dist_(a, b, key):
        if key == "loss":
            return abs(a - b)
        return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))

    outside = set()
    for rank, arms in enumerate(res):
        run = {"loss": 0.0, "grad": 0.0, "rs": 0.0}
        for i in range(steps):
            ref = arms["ref"][i]
            for key in run:
                run[key] = max(run[key], dist_(arms["emu"][i][key], ref[key], key))
                floor = 0.02 * abs(ref["loss"]) + 1e-3 if key == "loss" else 1e-3
                tol = 3.0 * run[key] + floor
                e_dev = dist_(arms["device"][i][key], ref[key], key)
                e_per = dist_(arms["per_rank"][i][key], ref[key], key)
                print(f"rank {rank} step {i} {key:4s}: device {e_dev:.3e}  emu {run[key]:.3e}  per-rank {e_per:.3e}  "
                      f"tol {tol:.3e}")
                assert e_dev <= tol, (rank, i, key, e_dev, tol)
                if i == 0 and e_per > tol:
                    outside.add(rank)
    # plain per-rank BatchNorm fails the same first-step check on both ranks
    assert outside == {0, 1}, f"per-rank BatchNorm passes every first-step check on rank(s) {sorted({0, 1} - outside)}"
    for a, b in zip(res[0]["device"], res[1]["device"]):
        assert np.array_equal(a["grad"], b["grad"]) and np.array_equal(a["rs"], b["rs"])


# ====================================================================================== 4. different sizes per rank
def _seeds_with_different_sizes():
    import random
    from yolov5_obb_b200.train_step import multi_scale_shape
    draws = {s: multi_scale_shape(S, 32, S, S, random.Random(s))[:2] for s in range(1, 40)}
    s0 = 1
    s1 = next(s for s in draws if draws[s] != draws[s0] and draws[s] != (S, S) and draws[s0] != (S, S))
    return s0, s1, draws[s0], draws[s1]


def _sizes_worker(rank, ws, seeds):
    from yolov5_obb_b200.train_step import TrainStep
    m = build_mirror("n", nc=15, seed=1).train().to(DEV)
    ts = TrainStep(m, batch_size=64, imgsz=S, multi_scale=True, seed=seeds[rank], sync_bn=True)
    names = {id(mod): n for n, mod in m.named_modules()}
    before = {n: host(torch.cat([b.running_mean, b.running_var])) for n, b in m.named_modules()
              if isinstance(b, torch.nn.BatchNorm2d)}
    imgs, tg = batch(seed=3 + rank)
    ts.step(imgs.to(DEV), tg.to(DEV))
    eng = m._last_train_engine
    lays = [dict(z=host(lay.z.view()), rec=host(lay.rec), mean=host(lay.mean), invstd=host(lay.invstd),
                 scale=host(lay.scale), shift=host(lay.shift), rs0=before[names[id(lay.mod.bn)]],
                 rs=host(torch.cat([lay.mod.bn.running_mean, lay.mod.bn.running_var]))) for lay in eng.conv_layers]
    return ts.last_shape, lays


def test_multi_scale_ranks_of_different_sizes_share_statistics():
    """One --multi-scale step in which the ranks draw different sizes.  Per BatchNorm layer: the summed record carries
    both ranks' pixel counts and their sums within the summation bound of fp64 sums over the union of both ranks' z maps;
    mean, invstd and the running statistics follow from it as y5obb_bn_finalize does (tests/bnref.py), and where the
    channel's |mean| / sigma <= 10 they match fp64 statistics of the union as the single-rank kernels do (beyond that the
    fp32 E[z^2] - E[z]^2 loses the variance, DESIGN.md section 7).  Both ranks hold the same statistics bit for bit."""
    s0, s1, hw0, hw1 = _seeds_with_different_sizes()
    (sh0, l0), (sh1, l1) = spawn(_sizes_worker, 2, (s0, s1))
    assert (sh0, sh1) == (hw0, hw1) and sh0 != sh1
    sms = _sms()
    worst, beyond = {}, 0

    def note(k, r):
        worst[k] = max(worst.get(k, 0.0), float(r))
        assert r <= 1.0, f"BN {li} (C {C}, {n0} + {n1} pixels) {k}: error {r:.3f} x its bound"

    mom1, momf = float(np.float32(1.0 - MOM)), float(np.float32(MOM))
    for li, (a, b) in enumerate(zip(l0, l1)):
        for k in ("rec", "mean", "invstd", "scale", "shift", "rs0", "rs"):
            assert np.array_equal(a[k], b[k]), f"BN {li}: {k} differs between the ranks"
        C = a["z"].shape[-1]
        za = torch.from_numpy(a["z"]).view(torch.bfloat16).reshape(-1, C)
        zb = torch.from_numpy(b["z"]).view(torch.bfloat16).reshape(-1, C)
        n0, n1 = za.shape[0], zb.shape[0]
        n = n0 + n1
        rec = torch.from_numpy(a["rec"])
        assert n0 != n1 and rec[2 * C].item() == n, f"BN {li}: the record's count is not {n0} + {n1}"
        x = torch.cat([za, zb]).double()
        d = max(stat_chain(n0, C, sms), stat_chain(n1, C, sms)) + 1
        s, q = rec[:C], rec[C:2 * C]
        note("sum", ((s - x.sum(0)).abs() / (gamma(d) * x.abs().sum(0)).clamp(min=1e-300)).max().item())
        note("sum of squares", ((q - (x * x).sum(0)).abs() / (gamma(d) * (x * x).sum(0)).clamp(min=1e-300)).max().item())
        m64, var64, iv64 = bnref.finalize_ref(s, q, n, EPS)
        mean, iv = torch.from_numpy(a["mean"]), torch.from_numpy(a["invstd"])
        assert torch.equal(mean, m64.float()), f"BN {li}: mean is not (float)(sum / n) of the summed record"
        note("invstd (ulp)", ((iv.double() - iv64).abs() / ulp32(iv64)).max().item())
        rm0, rv0 = [torch.from_numpy(t).double() for t in np.split(a["rs0"], 2)]
        rm, rv = [torch.from_numpy(t).double() for t in np.split(a["rs"], 2)]
        for key, got, new, old in (("running_mean", rm, mean.double(), rm0), ("running_var", rv, var64 * n / (n - 1.0), rv0)):
            want = mom1 * old + momf * new
            tol = 4 * U * (mom1 * old.abs() + momf * new.abs()) + ulp32(want)
            note(key, ((got - want).abs() / tol).max().item())
        mt = x.mean(0)
        sig = ((x - mt) ** 2).mean(0).sqrt()
        ok = mt.abs() <= 10 * sig
        beyond += int((~ok).sum())
        ivt = 1.0 / torch.sqrt(sig ** 2 + float(np.float32(EPS)))
        if ok.any():
            note("mean vs fp64", ((mean.double() - mt).abs() / (gamma(d) * x.abs().sum(0) / n + ulp32(mt)))[ok].max().item())
            note("invstd quality", ((iv.double() - ivt).abs() / ivt)[ok].max().item() / 2 ** -10)
    print(f"\n[sync-bn sizes] {hw0} and {hw1}: {len(l0)} layers; {beyond} channels beyond |mean| / sigma = 10; worst error / "
          f"bound {({k: f'{v:.3e}' for k, v in worst.items()})}")


# ============================================================================================== 5. graph capture
def _capture_worker(rank, ws):
    from yolov5_obb_b200.train_engine import TrainEngine
    m_p = build_mirror("n", nc=15, seed=1).train().to(DEV)
    m_s = copy.deepcopy(m_p)
    B = 2
    plain = TrainEngine(m_p, B, S, S, DEV)
    sync = TrainEngine(m_s, B, S, S, DEV, bn_group=dist.group.WORLD)
    assert sync.use_graph and sync.bn_rec is not None
    g = torch.Generator().manual_seed(0)
    n_steps = 5
    for k in range(n_steps):
        x = synth_tiles(B, S, seed=20 + k).to(DEV)
        grads = [torch.randn(o.shape, generator=g).to(DEV) * 1e-2 for o in plain.det_out]
        outs = []
        for eng in (plain, sync):
            det = [o.clone() for o in eng.forward(x, refresh=k > 0)]
            flat = eng.backward(grads).flat.clone()
            outs.append((det, flat))
        torch.cuda.synchronize()
        for a, b in zip(outs[0][0], outs[1][0]):
            assert torch.equal(a, b), f"step {k}: Detect logits differ"
        same_grads(grad_parts(host(outs[0][1]), m_p), grad_parts(host(outs[1][1]), m_s), f"step {k}")
    for a, b in zip(bn_state(m_p), bn_state(m_s)):
        assert torch.equal(a, b)
    captured = (len(sync._graphs), sync._bwd._graph is not None)
    return captured


def test_nccl_one_rank_sync_plans_capture_and_replay_bit_exact():
    """A one-rank NCCL group passed to TrainEngine: the forward's and the backward's all-reduces are captured in their
    CUDA graphs; five steps (eager, captured, replayed) equal the plain plans bit for bit."""
    (captured,) = spawn(_capture_worker, 1, backend="nccl")
    assert captured == (1, True)


# ================================================================================================== 6. fallback
def _fallback_pair(imgs, tg):
    """One TrainStep.step with sync_bn False and True: loss, gradient, activations, logits, running statistics."""
    from yolov5_obb_b200.train_step import TrainStep
    out = []
    for sync_bn in (False, True):
        m = build_mirror("n", nc=15, seed=1).train().to(DEV)
        ts = TrainStep(m, batch_size=64, imgsz=S, sync_bn=sync_bn)
        assert m.bn_group is None and not ts.sync_bn
        res = _run_identical(ts, m, imgs.to(DEV), tg.to(DEV), 1, lambda eng: host(eng._bwd.flat))
        assert m._last_train_engine.bn_group is None and m._last_train_engine.bn_rec is None
        out.append(res)
    return out


def _fallback_worker(rank, ws):
    return _fallback_pair(*batch())


def _same(pair):
    (sa, act_a, det_a, rs_a), (sb, act_b, det_b, rs_b) = pair
    assert np.array_equal(sa[0]["loss"], sb[0]["loss"])
    same_grads(sa[0]["flat"], sb[0]["flat"], "sync_bn=True fallback")
    for xa, xb in ((act_a, act_b), (det_a, det_b), (rs_a, rs_b)):
        assert all(np.array_equal(a, b) for a, b in zip(xa, xb))


def test_sync_bn_without_a_group_or_at_world_one_is_the_plain_step():
    assert not dist.is_initialized()
    _same(_fallback_pair(*batch()))
    (pair,) = spawn(_fallback_worker, 1)
    _same(pair)
