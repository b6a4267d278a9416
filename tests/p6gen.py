"""Seeded inputs of the P6 (models/hub/yolov5{n,s,m,l,x}6.yaml) goldens, shared by tests/golden/make_p6_golden.py (run on the
REFERENCE model) and the P6 tests (run on the oracle / the engine)."""
import numpy as np
import torch

from tests.lossgen import gaussian_label, synth_targets, PI

STRIDES = [8.0, 16.0, 32.0, 64.0]
_ANCH = torch.tensor([[19, 27, 44, 40, 38, 94], [96, 68, 86, 152, 180, 137], [140, 301, 303, 264, 238, 542],
                      [436, 615, 739, 380, 925, 792]]).float()
ANCHORS_GRID = _ANCH.view(4, 3, 2) / torch.tensor(STRIDES).view(4, 1, 1)   # Detect.anchors after yolo.py:124
LOSS_B, LOSS_H, LOSS_W = 2, 256, 320


def eval_input():
    """The seeded 1x3x128x192 image of the eval and train-mode goldens."""
    return torch.rand(1, 3, 128, 192, generator=torch.Generator().manual_seed(123))


def tta_input():
    """The seeded 1x3x256x320 image of the TTA golden: the 0.83 and 0.67 branches resample to a ragged size and pad to 64."""
    return torch.rand(1, 3, 256, 320, generator=torch.Generator().manual_seed(321))


def p6_targets(B, H, W, nt=40, nc=15, seed=0):
    """[nt + 8, 187] targets: nt DOTA-shaped ones (tests/lossgen.synth_targets, 8-300 px) and 8 boxes of 1150-1500 px, more than
    4x every P5 anchor (303 x 264 px at most) and within 4x of the P6 ones, so they match on P6 only."""
    t = synth_targets(B, nt, min(H, W), nc=nc, seed=seed)
    rng = np.random.default_rng(seed + 1000)
    big = np.zeros((8, 187), np.float32)
    big[:, 0] = rng.integers(0, B, 8)
    big[:, 1] = rng.integers(0, nc, 8)
    big[:, 2] = rng.uniform(0, W, 8)
    big[:, 3] = rng.uniform(0, H, 8)
    big[:, 4] = rng.uniform(1250, 1500, 8)
    big[:, 5] = big[:, 4] * rng.uniform(0.8, 1.0, 8)
    theta = (rng.integers(0, 180, 8) - 90) / 180 * PI
    big[:, 6] = theta
    for i in range(8):
        big[i, 7:] = gaussian_label(theta[i] * 180 / PI + 90)
    return np.concatenate([t, big])


def loss_preds(seed=0, no=200, scale=1.5):
    """Seeded Detect training outputs [B, 3, H / s, W / s, no] of the four levels."""
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(LOSS_B, 3, LOSS_H // int(s), LOSS_W // int(s), no, generator=g) * scale for s in STRIDES]


def loss_targets(seed=0):
    return torch.from_numpy(p6_targets(LOSS_B, LOSS_H, LOSS_W, seed=seed))
