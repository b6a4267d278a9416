"""CPU tests of whole-scene inference: tile geometry against the reference's own SplitSingle, and the CPU restatement of the
tile-merge chain (oracle/scene_ref.py) against the reference's own mergesingle (tests/golden/scene_golden.npz)."""
from pathlib import Path

import numpy as np
import pytest

from oracle import scene_ref
from yolov5_obb_b200.scene import split_origins, tile_geometry

G = np.load(Path(__file__).resolve().parent / "golden" / "scene_golden.npz")


def test_split_origins_match_reference_splitsingle():
    keys = [k for k in G.files if k.startswith("split/")]
    assert len(keys) >= 10
    for k in keys:
        H, W = map(int, k.split("/")[1].split("x"))
        assert split_origins(H, W, 1024, 200) == [tuple(o) for o in G[k].tolist()], k


def test_split_origins_refuses_gap_not_below_subsize():
    with pytest.raises(RuntimeError):
        split_origins(2000, 2000, 1024, 1024)


def test_tile_geometry_follows_val_rect_batching_and_letterbox():
    assert tile_geometry(1024, 0.5) == (1056, 16, 16.0)
    assert tile_geometry(1024, 0.0) == (1024, 0, 0.0)
    # an odd border: letterbox puts round(d - 0.1) on the top / left, scale_polys removes d
    assert tile_geometry(1001, 0.5) == (1024, 11, 11.5)


def _tiles():
    org, polys, rows, counts = G["merge/origins"], G["merge/polys"], G["merge/rows"], G["merge/counts"]
    return [(int(l), int(u), polys[t, :counts[t]], rows[t, :counts[t], 5], rows[t, :counts[t], 6].astype(np.int64))
            for t, (l, u) in enumerate(org.tolist())]


def test_merge_restatement_matches_reference_mergesingle():
    got = scene_ref.merge(_tiles(), 15, 0.2)
    want = G["merge/merged"]
    assert got.shape == want.shape
    assert np.array_equal(got, want)
    # the inputs carry exact rounding ties of round(x, 1) and detections repeated across tile overlaps
    raw = np.concatenate([p.reshape(-1) for _, _, p, _, _ in _tiles()]).astype(np.float64)
    assert np.any(np.abs(raw * 10 - np.floor(raw * 10) - 0.5) == 0)
    assert want.shape[0] < G["merge/counts"].sum()


def test_task1_text_matches_reference_mergesingle():
    names = [str(n) for n in G["merge/names"]]
    text = scene_ref.task1_lines(G["merge/merged"], "P0000", names)
    for c in range(15):
        k = f"merge/text/{c}"
        if k in G.files:
            assert text[f"Task1_{names[c]}.txt"] == str(G[k]), names[c]
