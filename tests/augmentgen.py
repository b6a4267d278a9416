"""Seeded cached datasets for the training-augmentation tests: structured, compressible uint8 BGR images whose longest side
is img_size (load_image_label's cached form), with DOTA-like labels [n, 9] fp32 (cls, 4 corner points), some crossing the
image edges, some degenerate (zero area, repeated points), and some images without labels."""
import numpy as np

# data/hyps/obb/hyp.finetune_dota.yaml (augmentation and target keys)
HYP_DOTA = dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=180.0, translate=0.1, scale=0.25, shear=0.0, perspective=0.0,
                flipud=0.5, fliplr=0.5, mosaic=0.75, mixup=0.1, copy_paste=0.0, cls_theta=180, csl_radius=2.0)


def synth_image(rng, h, w):
    y, x = np.mgrid[0:h, 0:w]
    f = rng.uniform(0.01, 0.08, 3)
    ph = rng.uniform(0, 6.28, 3)
    img = np.stack([127.5 + 127.5 * np.sin(f[c] * (x + (c + 1) * y) + ph[c]) for c in range(3)], -1)
    for _ in range(int(rng.integers(2, 6))):  # flat blocks: saturated and grey colours
        x0, y0 = int(rng.integers(0, w - 8)), int(rng.integers(0, h - 8))
        img[y0:y0 + int(rng.integers(8, 64)), x0:x0 + int(rng.integers(8, 64))] = rng.integers(0, 256, 3)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def synth_labels(rng, h, w, n, nc=15):
    if n == 0:
        return np.zeros((0, 9), np.float32)
    cx, cy = rng.uniform(-0.1 * w, 1.1 * w, n), rng.uniform(-0.1 * h, 1.1 * h, n)
    lw, lh = rng.uniform(2, 0.4 * w, n), rng.uniform(2, 0.2 * h, n)
    th = rng.uniform(-np.pi, np.pi, n)
    c, s = np.cos(th), np.sin(th)
    pts = []
    for dx, dy in ((-1, -1), (1, -1), (1, 1), (-1, 1)):
        pts += [cx + dx * lw / 2 * c - dy * lh / 2 * s, cy + dx * lw / 2 * s + dy * lh / 2 * c]
    P = np.stack(pts, 1)
    P[::7, 2:4] = P[::7, 0:2]          # a repeated corner
    P[3::9, 4:] = P[3::9, :4]          # zero area
    P = np.round(P, 1)                 # labelTxt coordinates are decimal
    cls = rng.integers(0, nc, n).astype(np.float64)
    return np.concatenate([cls[:, None], P], 1).astype(np.float32)


def synth_dataset(n_images, S, seed, max_labels=20):
    rng = np.random.default_rng(seed)
    images, labels = [], []
    for i in range(n_images):
        short = int(rng.integers(S // 2, S + 1))
        h, w = (S, short) if i % 2 else (short, S)
        images.append(synth_image(rng, h, w))
        labels.append(synth_labels(rng, h, w, 0 if i % 5 == 4 else int(rng.integers(1, max_labels + 1))))
    return images, labels
