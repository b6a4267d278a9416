"""Optimizer-step timing (dev tool): the fused Adam + EMA step (train_ops.FusedAdamEMA, one launch) against torch.optim.Adam's
foreach step + ModelEMA.update, the step train.py --adam runs, with the fused SGD + EMA step (train_ops.FusedSGDEMA) as a
reference point.  Parameter sets of yolov5s and yolov5m with nc = 15, the reference's three parameter groups, gradients as
views of one flat buffer (as the backward plan hands them over).  Each figure is the CUDA-event mean per step over `iters`
steps after `warmup` steps; the three steps are timed in turn, `reps` rounds, and the median round is reported with the
range of all rounds.  Per model:
  param_elems / buffer_elems   parameter elements (optimizer + EMA) and floating-point buffer elements (EMA only)
  adam_bytes                   36 B per parameter element (p, g, exp_avg, exp_avg_sq, ema read; p, moments, ema written)
                               + 12 B per buffer element; adam_fused_GBps = adam_bytes / adam_fused_ms
  sgd_bytes                    28 B per parameter element + 12 B per buffer element
and the card's name and power limit, read in the same run.
python tools/time_optimizer.py [iters] [warmup] [reps]"""
import copy
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from tests.modelgen import build_mirror  # noqa: E402
from yolov5_obb_b200.train_ops import FusedAdamEMA, FusedSGDEMA  # noqa: E402
from yolov5_obb_b200.train_step import HYP_FINETUNE_DOTA, ModelEMA, param_groups  # noqa: E402

BETAS, EPS, WD, LR = (HYP_FINETUNE_DOTA["momentum"], 0.999), 1e-8, HYP_FINETUNE_DOTA["weight_decay"], 1e-4


def event_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def flat_grads(model, dev, seed):
    params = list(model.parameters())
    flat = torch.randn(sum(p.numel() for p in params), generator=torch.Generator(device=dev).manual_seed(seed), device=dev)
    out, o = {}, 0
    for p in params:
        out[p] = flat[o:o + p.numel()].view_as(p)
        o += p.numel()
    return out


def run(size, dev, iters, warmup, reps):
    base = build_mirror(size, nc=15, seed=0).to(dev).train()
    n_par = sum(p.numel() for p in base.parameters())
    pnames = {n for n, _ in base.named_parameters()}
    n_buf = sum(v.numel() for k, v in base.state_dict().items() if k not in pnames and v.dtype.is_floating_point)

    m_fa = copy.deepcopy(base)
    ema_fa = ModelEMA(m_fa)
    fa = FusedAdamEMA(m_fa, param_groups(m_fa), flat_grads(m_fa, dev, 1), ema_fa.ema, weight_decay=WD)

    m_ta = copy.deepcopy(base)
    ema_ta = ModelEMA(m_ta)
    g0, g1, g2 = param_groups(m_ta)
    opt = torch.optim.Adam(g0, lr=LR, betas=BETAS, foreach=True)
    opt.add_param_group({"params": g1, "weight_decay": WD})
    opt.add_param_group({"params": g2})
    for p, g in flat_grads(m_ta, dev, 1).items():
        p.grad = g

    m_fs = copy.deepcopy(base)
    ema_fs = ModelEMA(m_fs)
    fs = FusedSGDEMA(m_fs, param_groups(m_fs), flat_grads(m_fs, dev, 1), ema_fs.ema, weight_decay=WD)

    def fused_adam():
        ema_fa.updates += 1
        fa.step((LR, LR, LR), BETAS, EPS, ema_fa.decay(ema_fa.updates))

    def torch_adam():
        opt.step()
        ema_ta.update(m_ta)

    def fused_sgd():
        ema_fs.updates += 1
        fs.step((LR, LR, LR), BETAS[0], ema_fs.decay(ema_fs.updates))

    arms = {"adam_fused": fused_adam, "adam_torch": torch_adam, "sgd_fused": fused_sgd}
    times = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            times[k].append(event_ms(fn, iters, warmup))
    out = {"param_elems": n_par, "buffer_elems": n_buf, "adam_bytes": 36 * n_par + 12 * n_buf, "sgd_bytes": 28 * n_par + 12 * n_buf}
    for k, v in times.items():
        out[f"{k}_ms"] = round(statistics.median(v), 4)
        out[f"{k}_ms_range"] = [round(min(v), 4), round(max(v), 4)]
    out["adam_fused_GBps"] = round(out["adam_bytes"] / out["adam_fused_ms"] / 1e6, 1)
    out["sgd_fused_GBps"] = round(out["sgd_bytes"] / out["sgd_fused_ms"] / 1e6, 1)
    out["adam_speedup"] = round(out["adam_torch_ms"] / out["adam_fused_ms"], 2)
    return out


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
    if not torch.cuda.is_available():
        raise SystemExit("time_optimizer.py needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda:0")
    res = {"card": card, "iters": iters, "warmup": warmup, "reps": reps, "nc": 15}
    for size in ("s", "m"):
        res[f"yolov5{size}"] = run(size, dev, iters, warmup, reps)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
