"""Input and golden layout of the test-time-augmentation goldens, shared by tests/golden/make_tta_golden.py (run on the
REFERENCE model) and the tests (run on the oracle / the engine).

The whole augmented output would be 4 MB per model, so tta_golden.npz keeps, per model:
  box     columns 0-3 (the de-scaled, de-flipped x y w h) of every row;
  rows    every column of every ROW_STEP-th row (all three branches, every level, anchor and class / angle bin column);
  rowsum  the fp64 sum of every row's columns (each element enters some check);
and the fp64 sum of the input, which confirms that tta_input() regenerated the same image."""
import numpy as np
import torch

ROW_STEP = 53   # prime, so that the sampled rows walk through anchors, grid positions and levels


def tta_input():
    """The seeded 2x3x128x160 image: both scaled branches resample to a ragged size and pad."""
    return torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(321))


def pieces(pred: np.ndarray) -> dict:
    return {"box": pred[..., :4].copy(), "rows": pred[:, ::ROW_STEP].copy(),
            "rowsum": pred.astype(np.float64).sum(-1)}
