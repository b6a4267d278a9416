"""Host geometry of --multi-scale training (train_step.multi_scale_shape) against the restatement of train.py:314-318."""
import math
import random

from oracle import multiscale_ref
from yolov5_obb_b200.train_step import multi_scale_max_shape, multi_scale_shape


class _Fixed:
    """A generator whose every draw is `v` (walks every drawable size)."""

    def __init__(self, v):
        self.v = v

    def randrange(self, lo, hi):
        assert lo <= self.v < hi
        return self.v


def test_every_imgsz_and_every_drawable_size():
    gs, ceil_up = 32, 0
    for imgsz in range(64, 2049, 32):
        for v in range(int(imgsz * 0.5), int(imgsz * 1.5 + gs)):
            for H, W in ((imgsz, imgsz), (imgsz, imgsz // 2 // gs * gs or gs)):
                got = multi_scale_shape(imgsz, gs, H, W, _Fixed(v))
                ns, ratio = multiscale_ref.new_shape(multiscale_ref.draw_size(_Fixed(v), imgsz, gs), gs, (H, W))
                want = (H, W, 1.0) if ns is None else (ns[0], ns[1], ratio)
                assert got == want and type(got[2]) is float, (imgsz, v, H, W, got, want)
        # the fp64 ceil that rounds one grid step up (square batches, counted once per size)
        for sz in range(int(imgsz * 0.5) // gs * gs, int(imgsz * 1.5 + gs), gs):
            if sz >= int(imgsz * 0.5) and sz != imgsz and multi_scale_shape(imgsz, gs, imgsz, imgsz, _Fixed(sz))[0] == sz + gs:
                ceil_up += 1
    assert ceil_up == 69
    assert multi_scale_shape(800, 32, 800, 800, _Fixed(448))[:2] == (480, 480)


def test_max_shape_covers_every_draw():
    for imgsz in (160, 800, 1024):
        hmax, wmax = multi_scale_max_shape(imgsz, 32, imgsz, imgsz)
        seen = {multi_scale_shape(imgsz, 32, imgsz, imgsz, _Fixed(v))[:2]
                for v in range(int(imgsz * 0.5), int(imgsz * 1.5 + 32))}
        assert (hmax, wmax) == max(seen)
    assert multi_scale_max_shape(1024, 32, 1024, 1024) == (1536, 1536)
    assert multi_scale_max_shape(160, 32, 160, 160) == (256, 256)


def test_seeded_generator_gives_the_reference_draws():
    """TrainStep's own generator (seed=None: train.py's init_seeds(1 + RANK), RANK -1 without DDP) against random.Random
    under the reference expression; the module-level `random` is not touched."""
    from tests.modelgen import build_mirror
    from yolov5_obb_b200.train_step import TrainStep
    m = build_mirror("n", nc=15, seed=0).train()
    for seed in (None, 1, 7):
        rng = random.Random(0 if seed is None else seed)
        want = []
        for _ in range(1000):
            sz = multiscale_ref.draw_size(rng, 1024, 32)
            ns, _ = multiscale_ref.new_shape(sz, 32, (1024, 1024))
            want.append((1024, 1024) if ns is None else tuple(ns))
        ts = TrainStep(m, batch_size=64, imgsz=1024, ema=False, seed=seed)   # multi_scale=False: no device needed
        state = random.getstate()
        got = [multi_scale_shape(ts.imgsz, ts.gs, 1024, 1024, ts.rng)[:2] for _ in range(1000)]
        assert got == want and random.getstate() == state
    # 33 sizes for imgsz 1024: 512 ... 1536
    sizes = {multi_scale_shape(1024, 32, 1024, 1024, _Fixed(v))[0] for v in range(512, 1568)}
    assert sorted(sizes) == list(range(512, 1537, 32)) and len(sizes) == 33
    assert math.isclose(multi_scale_shape(1024, 32, 1024, 1024, _Fixed(640))[2], 0.625)
