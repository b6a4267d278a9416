"""SyncBatchNorm in the training plans (train.py --sync-bn): what the per-layer collectives cost.

  * collectives: per training step, one all-reduce per BatchNorm layer in the forward plan (its [sum | sum of squares |
    count] record, 2C + 1 doubles) and one per live BatchNorm backward (2C doubles); counted from the model for each size
    (the count and bytes do not depend on batch or image size).
  * one GPU: the plain plans against the sync plans forced onto a one-rank NCCL group (TrainEngine(bn_group=...)), forward +
    backward with their CUDA graphs (the collectives captured), timed alternately with CUDA events; the mean time per
    collective is the difference over the number of collectives.  A one-rank NCCL all-reduce moves no data, so this is the
    launch and synchronisation cost of the collectives inside the graphs.
  * N ranks (N GPUs): TrainStep.step with sync_bn False / True, one rank per GPU over NCCL; not measured with one GPU.
The card's name and power limit are read in the same run.  Prints one JSON line.
usage: python tools/time_sync_bn.py [steps=20] [rounds=3] [B=8] [imgsz=1024] [sizes=s,m]"""
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from tests.modelgen import build_mirror
from tests.tilegen import synth_tiles


def collectives(size, B=16, S=1024):
    """(number, bytes) of the all-reduces of one training step of yolov{size} (every layer trainable)."""
    from yolov5_obb_b200.yolo import Model
    cs = [mod.num_features for mod in Model(f"yolov5{size}.yaml", nc=15).modules() if isinstance(mod, torch.nn.BatchNorm2d)]
    return dict(model=f"yolov5{size}", batch=B, imgsz=S, forward=len(cs), backward=len(cs),
                bytes_forward=8 * sum(2 * c + 1 for c in cs), bytes_backward=8 * sum(2 * c for c in cs))


def one_gpu(size, B, S, steps, rounds, dev):
    from yolov5_obb_b200.train_engine import TrainEngine
    m_p = build_mirror(size, nc=15, seed=0).train().to(dev)
    m_s = build_mirror(size, nc=15, seed=0).train().to(dev)
    engs = dict(plain=TrainEngine(m_p, B, S, S, dev), sync=TrainEngine(m_s, B, S, S, dev, bn_group=dist.group.WORLD))
    x = synth_tiles(B, S, seed=1).to(dev)
    g = torch.Generator(device=dev).manual_seed(0)
    grads = [1e-3 * torch.randn(o.shape, device=dev, generator=g) for o in engs["plain"].det_out]
    times = {k: [] for k in engs}

    def step(eng):
        eng.forward(x, refresh=True)
        eng.backward(grads)

    for k, eng in engs.items():
        for _ in range(3):    # eager, captured, replayed
            step(eng)
    torch.cuda.synchronize()
    for _ in range(rounds):
        for k, eng in engs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                step(eng)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / steps)
    n = len(engs["sync"].conv_layers) + sum(1 for t, _ in engs["sync"]._bwd.steps if t == "bn_allreduce")
    med = {k: statistics.median(v) for k, v in times.items()}
    return dict(model=f"yolov5{size}", batch=B, imgsz=S, ms_plain=med["plain"], ms_sync=med["sync"],
                ms_plain_range=[min(times["plain"]), max(times["plain"])],
                ms_sync_range=[min(times["sync"]), max(times["sync"])], collectives=n,
                us_per_collective=1e3 * (med["sync"] - med["plain"]) / n)


def _rank(rank, ws, port, size, B, S, steps, q):
    import time
    from tests.lossgen import synth_targets
    from yolov5_obb_b200.train_step import TrainStep
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=ws, device_id=dev)
    try:
        imgs = synth_tiles(B, S, seed=1 + rank).to(dev)
        tg = torch.from_numpy(synth_targets(B, 24 * B, S, nc=15, seed=2 + rank)).to(dev)
        res = {}
        for sync_bn in (False, True):
            m = build_mirror(size, nc=15, seed=0).train().to(dev)
            ts = TrainStep(m, batch_size=64, imgsz=S, sync_bn=sync_bn)
            for _ in range(3):
                ts.step(imgs, tg)
            torch.cuda.synchronize()
            dist.barrier()
            t0 = time.perf_counter()
            for _ in range(steps):
                ts.step(imgs, tg)
            torch.cuda.synchronize()
            res["sync" if sync_bn else "plain"] = (time.perf_counter() - t0) * 1e3 / steps
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def n_ranks(size, B, S, steps, ws):
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank, args=(r, ws, port, size, B, S, steps, q)) for r in range(ws)]
    for p in procs:
        p.start()
    try:
        res = [q.get(timeout=1800) for _ in range(ws)]
    finally:
        for p in procs:
            p.join(60)
            if p.is_alive():
                p.kill()
                p.join()
    return dict(model=f"yolov5{size}", ranks=ws, batch_per_rank=B, imgsz=S,
                ms_plain=max(r["plain"] for _, r in res), ms_sync=max(r["sync"] for _, r in res))


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    B = int(sys.argv[3]) if len(sys.argv) > 3 else 8
    S = int(sys.argv[4]) if len(sys.argv) > 4 else 1024
    sizes = sys.argv[5].split(",") if len(sys.argv) > 5 else ["s", "m"]
    out = dict(collectives_per_step=[collectives(sz) for sz in ("s", "m")])
    if not torch.cuda.is_available():
        out.update(card="no GPU", one_gpu="not measured", n_ranks="not measured")
        print(json.dumps(out))
        return
    out["card"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                 capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda:0")
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=os.environ.get("MASTER_PORT", "29517"))
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=dev)
    try:
        out["one_gpu"] = [one_gpu(sz, B, S, steps, rounds, dev) for sz in sizes]
    finally:
        dist.destroy_process_group()
    ws = torch.cuda.device_count()
    out["n_ranks"] = [n_ranks(sz, B, S, steps, ws) for sz in sizes] if ws > 1 else f"not measured ({ws} GPU)"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
