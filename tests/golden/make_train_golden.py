"""Golden vectors from the REFERENCE model in TRAIN mode (models/yolo.py Model: batch-statistic BatchNorm, raw Detect
outputs, autograd backward as train.py:324-333 drives it) - run where the reference checkout exists:
    python tests/golden/make_train_golden.py
Writes train_golden.npz for yolov5n (nc=15, torch seed 0, tests/modelgen.seeded_state): the three training outputs on a
seeded 2x3x64x96 batch; for every parameter gradient of a fixed linear functional of them its fp64 norm, its fp64 dot
product with a seeded probe vector and its first 64 elements (the file stays small); the BatchNorm running statistics
after the step."""
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import ref_import  # noqa: E402

ref_import.setup()
sys.path.insert(0, str(HERE.parents[1]))
from models.yolo import Model  # noqa: E402  (the reference)
from tests.modelgen import seeded_state  # noqa: E402


def main():
    torch.manual_seed(0)
    m = Model("models/yolov5n.yaml", ch=3, nc=15)
    seeded_state(m, 0).train()
    g = torch.Generator().manual_seed(321)
    x = torch.rand(2, 3, 64, 96, generator=g)
    outs = m(x)
    G = [torch.randn(o.shape, generator=g) * 0.05 for o in outs]
    sum((o * gg).sum() for o, gg in zip(outs, G)).backward()
    out = {"x": x.numpy()}
    for l, (o, gg) in enumerate(zip(outs, G)):
        out[f"out{l}"] = o.detach().numpy()
        out[f"G{l}"] = gg.numpy()
    names = []
    for i, (n, p) in enumerate(m.named_parameters()):
        names.append(n)
        gflat = p.grad.double().flatten()
        probe = torch.randn(gflat.numel(), generator=torch.Generator().manual_seed(1000 + i), dtype=torch.float64)
        out[f"grad/{n}"] = np.concatenate([[gflat.norm().item(), (gflat * probe).sum().item()], gflat[:64].numpy()])
    out["names"] = np.array(names)
    for n, b in m.named_buffers():
        if n.endswith("running_mean") or n.endswith("running_var"):
            out[f"buf/{n}"] = b.numpy()
    np.savez_compressed(HERE / "train_golden.npz", **out)
    print(len(names), "parameter gradients;", [tuple(o.shape) for o in outs])


if __name__ == "__main__":
    main()
