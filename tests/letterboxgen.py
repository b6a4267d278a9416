"""Seeded source images for the letterbox tests (decoded uint8 [H, W, 3] BGR arrays, as cv2.imread returns them)."""
import numpy as np

# (h, w) of the golden set at img_size 128: fractional shrink, exact 2x, 3x, 4x, no resize, enlargement, extreme aspect ratios
GOLDEN_SIZES = [(300, 400), (97, 211), (256, 256), (384, 384), (512, 300), (128, 128), (100, 100), (640, 61), (33, 500),
                (129, 127), (255, 256)]
GOLDEN_IMG_SIZE = 128
GOLDEN_BATCH = 3
GOLDEN_PAD = 0.5
# the golden keeps every reference image as a SHA-256; these keep their bytes too, for the device tests: LoadImages items
# (fractional shrink, enlargement, exact 2x, 3x, extreme aspect ratio) and two whole rect batches
GOLDEN_FULL_DETECT = (0, 1, 2, 3, 7)
GOLDEN_FULL_RECT_BATCHES = (0, 2)


def synth_image(h: int, w: int, seed: int) -> np.ndarray:
    """Noise over a smooth ramp: every resampling tap matters and no two channels agree."""
    rng = np.random.default_rng(seed)
    ramp = (np.arange(h)[:, None, None] * 3 + np.arange(w)[None, :, None] * 5 + np.arange(3)[None, None, :] * 70) % 256
    noise = rng.integers(0, 256, (h, w, 3))
    return np.where(rng.random((h, w, 1)) < 0.7, noise, ramp).astype(np.uint8)


def golden_images():
    return [synth_image(h, w, 100 + i) for i, (h, w) in enumerate(GOLDEN_SIZES)]


def synth_polys(h: int, w: int, n: int, seed: int) -> np.ndarray:
    """n label polygons [n, 8] inside an h x w image (rotated rectangles)."""
    rng = np.random.default_rng(seed)
    c = rng.uniform([0.2 * w, 0.2 * h], [0.8 * w, 0.8 * h], (n, 2))
    wh = rng.uniform(0.05, 0.15, (n, 2)) * min(h, w)
    a = rng.uniform(-np.pi / 2, np.pi / 2, n)
    ux = np.stack([np.cos(a), np.sin(a)], 1) * wh[:, :1]
    uy = np.stack([-np.sin(a), np.cos(a)], 1) * wh[:, 1:]
    return np.concatenate([c + ux + uy, c - ux + uy, c - ux - uy, c + ux - uy], 1)
