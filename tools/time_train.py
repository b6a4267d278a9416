"""Phase timing of one training step (forward / loss / backward / optimiser+EMA) with CUDA events (debug aid).
usage: python tools/time_train.py [size=m] [B=8] [imgsz=1024] [steps=5]"""
import sys, time, torch
from tests.modelgen import build_mirror
from tests.tilegen import synth_tiles
from tests.lossgen import synth_targets
from yolov5_obb_b200.train_step import TrainStep

size = sys.argv[1] if len(sys.argv) > 1 else "m"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 8
S = int(sys.argv[3]) if len(sys.argv) > 3 else 1024
steps = int(sys.argv[4]) if len(sys.argv) > 4 else 5
warm = int(sys.argv[5]) if len(sys.argv) > 5 else 3
dev = "cuda:0"
m = build_mirror(size, nc=15, seed=0).train().to(dev)
ts = TrainStep(m, batch_size=64)
imgs = synth_tiles(B, S, seed=1).to(dev)
tg = torch.from_numpy(synth_targets(B, 24 * B, S, nc=15, seed=2)).to(dev)
ev = lambda: torch.cuda.Event(enable_timing=True)
for it in range(warm + steps):
    e = [ev() for _ in range(5)]
    t0 = time.perf_counter()
    e[0].record()
    pred = m(imgs)
    e[1].record()
    loss, items = ts.compute_loss(pred, tg)
    e[2].record()
    loss.backward()
    e[3].record()
    ts.optimizer.step(); ts.optimizer.zero_grad(set_to_none=True); ts.ema.update(m)
    e[4].record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3
    if it >= warm:
        d = [e[i].elapsed_time(e[i + 1]) for i in range(4)]
        print(f"step {it}: fwd {d[0]:.2f} loss {d[1]:.2f} bwd {d[2]:.2f} opt+ema {d[3]:.2f} total {sum(d):.2f} ms (wall {wall:.2f})  "
              f"{B / sum(d) * 1e3:.1f} img/s  loss {loss.item():.4f}", flush=True)
eng = m._last_train_engine
print("fwd flops %.3g  bwd flops %.3g  mem %.2f GB" % (eng.flops, eng._bwd.flops, torch.cuda.max_memory_allocated() / 2**30))

# per-kernel-kind device times of one more step (events around every launch; serialises nothing but adds gaps)
eng.prof = {}
eng._bwd.prof = {}
pred = m(imgs)
loss, items = ts.compute_loss(pred, tg)
loss.backward()
torch.cuda.synchronize()
for title, prof in (("forward", eng.prof), ("backward", eng._bwd.prof)):
    tot = sum(sum(v) for v in prof.values())
    print(title, f"{tot:.2f} ms:", "  ".join(f"{k} {sum(v):.2f} (x{len(v)})" for k, v in sorted(prof.items(), key=lambda kv: -sum(kv[1]))))
# the ten slowest conv / wgrad / dgrad launches with their shapes
desc = lambda l: f"{l.x.C}->{l.z.C} k{l.mod.conv.kernel_size[0]} s{l.mod.conv.stride[0]} {l.z.H}x{l.z.W}"
top = sorted(zip(eng.prof["conv"], eng.conv_layers), key=lambda t: -t[0])[:8]
print("slowest fwd convs:", "; ".join(f"{t*1e3:.0f}us {desc(l)} ({l.conv.info()['flops']/t/1e9:.0f} TF/s)" for t, l in top))
parts = eng._bwd.conv_parts
nd = len(eng._bwd.det_parts)
wg = eng._bwd.prof["wgrad"][nd:]   # the first are the Detect levels'
top = sorted(zip(wg, parts), key=lambda t: -t[0])[:8]
print("slowest wgrads:", "; ".join(f"{t*1e3:.0f}us {desc(p['lay'])} ({p['lay'].conv.info()['flops']/t/1e9:.0f} TF/s)" for t, p in top))
dg = eng._bwd.prof["dgrad"][nd:]
dl = []
for p in parts:  # stride-2 layers launch four parity-class convs
    n = 1 if "dgrad_wp" in p else (4 if "dgrad_s2" in p else 0)
    if n:
        dl.append((sum(dg[:n]), p))
        dg = dg[n:]
top = sorted(dl, key=lambda t: -t[0])[:8]
print("slowest dgrads:", "; ".join(f"{t*1e3:.0f}us {desc(p['lay'])} ({p['lay'].conv.info()['flops']/t/1e9:.0f} TF/s)" for t, p in top))
