"""Seeded inputs of the validation-loss golden (tests/golden/make_valloss_golden.py) and its tests: two batches of 2 uint8
images of 256 x 320 with [nt, 187] targets, and the model settings."""
import torch

from tests.lossgen import synth_targets
from tests.tilegen import synth_tiles

SIZES = ("n", "s")
OBJ_BIAS = -2.0        # raised Detect obj / cls biases (tests/modelgen.seeded_state): the obj BCE is not all near zero
B, H, W, NT = 2, 256, 320, 12
N_BATCHES = 2
HYP_IMGSZ = 320        # train.py:249-252 scales hyp['obj'] by (imgsz / 640) ** 2


def batch(i: int):
    """(uint8 images [B, 3, H, W], fp32 targets [NT, 187] in pixels) of batch i."""
    im = synth_tiles(B, W, seed=70 + i)[:, :, :H, :W].contiguous()
    tg = torch.from_numpy(synth_targets(B, NT, H, nc=15, seed=70 + i))
    return im, tg
