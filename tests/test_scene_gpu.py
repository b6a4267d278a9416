"""GPU tests of whole-scene inference (yolov5_obb_b200/scene.py, csrc/scene.cu): the tile input kernel against the stem layout
pass on tiles built in torch, the merge kernel against the reference's mergesingle (tests/golden/scene_golden.npz) and the CPU
restatement (oracle/scene_ref.py), SceneDetector against a composition of the existing public calls, and the refusals."""
import types
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import scene_ref
from tests.scenegen import tile_rows
from yolov5_obb_b200 import _lib
from yolov5_obb_b200.scene import SceneDetector, merge_tiles, split_origins, tile_geometry

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
G = np.load(Path(__file__).resolve().parent / "golden" / "scene_golden.npz")


def _scene(H, W, seed):
    from tests.tilegen import synth_tiles
    side = max(H, W) + (-max(H, W)) % 32
    return synth_tiles(1, side, seed)[0, :, :H, :W].permute(1, 2, 0).contiguous()   # HWC, read as BGR


def _torch_tiles(scene, origins, subsize, size, border):
    """ImgSplit crop + zero padding, letterbox border of 114, BGR -> RGB, NCHW: the PNG route restated in torch."""
    H, W = scene.shape[:2]
    out = torch.full((len(origins), 3, size, size), 114, dtype=torch.uint8)
    for t, (left, up) in enumerate(origins):
        tile = torch.zeros((subsize, subsize, 3), dtype=torch.uint8)
        crop = scene[up:up + subsize, left:left + subsize]
        tile[:crop.shape[0], :crop.shape[1]] = crop
        out[t, :, border:border + subsize, border:border + subsize] = tile.flip(2).permute(2, 0, 1)
    return out


@pytest.mark.parametrize("H,W", [(1700, 2300), (900, 700), (1024, 1024)])
@pytest.mark.parametrize("pad", [0.5, 0.0])
def test_tile_input_equals_stem_layout_of_torch_tiles(H, W, pad):
    L = _lib.lib()
    scene = _scene(H, W, 1)
    origins = split_origins(H, W)
    size, border, _ = tile_geometry(1024, pad)
    T = len(origins)
    got = torch.zeros((T, size // 2, size // 2 + 2, 16), dtype=torch.bfloat16, device=DEV)
    want = torch.zeros_like(got)
    sd = scene.to(DEV)
    org = torch.tensor(origins, dtype=torch.int32, device=DEV)
    st = _lib.stream_ptr(torch.device(DEV))
    _lib.check(L.y5obb_scene_tiles_s2d_u8(sd.data_ptr(), H, W, org.data_ptr(), T, 1024, size, border, got.data_ptr(), 1, st),
               "y5obb_scene_tiles_s2d_u8")
    tiles = _torch_tiles(scene, origins, 1024, size, border).to(DEV)
    _lib.check(L.y5obb_stem_s2d_u8(tiles.data_ptr(), want.data_ptr(), T, size, size, 1, st), "y5obb_stem_s2d_u8")
    assert torch.equal(got, want)


def _device_polys(rows, counts, pad):
    """rbox2poly + scale_polys through the existing public calls, per tile -> the oracle's input."""
    from yolov5_obb_b200.rboxs_utils import rbox2poly, scale_polys
    out = []
    for t in range(rows.shape[0]):
        r = rows[t, :int(counts[t])]
        poly = rbox2poly(r[:, :5])
        scale_polys((1056, 1056), poly, (1024, 1024), ratio_pad=((1.0, 1.0), (pad, pad)))
        out.append((poly.cpu().numpy(), r[:, 5].cpu().numpy(), r[:, 6].long().cpu().numpy()))
    return out


def test_merge_equals_reference_mergesingle():
    rows = torch.from_numpy(G["merge/rows"]).to(DEV)
    counts = torch.from_numpy(G["merge/counts"]).to(DEV)
    org = torch.from_numpy(G["merge/origins"]).to(DEV)
    for t, (p, _, _) in enumerate(_device_polys(rows, counts, 16.0)):   # theta = 0: rbox2poly is exact on any device
        assert np.array_equal(p, G["merge/polys"][t, :G["merge/counts"][t]])
    got = merge_tiles(rows, counts, org, 15, 16.0, 0.2).rows.cpu()
    assert torch.equal(got, torch.from_numpy(G["merge/merged"]))


def test_merge_equals_restatement_on_25_full_tiles(tmp_path):
    origins, rows_np, counts_np = tile_rows(4000, 4000, 40000, nc=15, seed=5)
    assert origins.shape[0] == 25 and (counts_np == 1500).all()
    rows, counts, org = torch.from_numpy(rows_np).to(DEV), torch.from_numpy(counts_np).to(DEV), torch.from_numpy(origins).to(DEV)
    res = merge_tiles(rows, counts, org, 15, 16.0, 0.2)
    tiles = [(int(l), int(u)) + d for (l, u), d in zip(origins.tolist(), _device_polys(rows, counts, 16.0))]
    want = scene_ref.merge(tiles, 15, 0.2)
    assert torch.equal(res.rows.cpu(), torch.from_numpy(want))
    assert sorted(res.per_class()) == sorted(set(want[:, 0].astype(int).tolist()))
    names = [f"class{c}" for c in range(15)]
    res.write_task1(tmp_path, "P0001", names)
    for fname, text in scene_ref.task1_lines(want, "P0001", names).items():
        assert (tmp_path / fname).read_text() == text


def test_merge_zero_area_polygons_suppress_as_in_c():
    """Zero-area polygons with overlapping axis-aligned boxes: polyiou's 0 / 0 is nan in C, which suppresses."""
    rows = torch.zeros((1, 8, 7))
    rows[0, :4] = torch.tensor([[100.0, 100.0, 20.0, 0.0, 0.5, 0.9, 0.0], [100.0, 100.0, 20.0, 0.0, 0.5, 0.8, 0.0],
                                [101.0, 100.0, 20.0, 0.0, 0.5, 0.7, 0.0], [300.0, 300.0, 40.0, 20.0, 0.3, 0.6, 0.0]])
    counts = torch.tensor([4])
    res = merge_tiles(rows.to(DEV), counts.to(DEV), torch.zeros((1, 2), dtype=torch.int32, device=DEV), 1, 16.0, 0.2)
    tiles = [(0, 0) + d for d in _device_polys(rows.to(DEV), counts, 16.0)]
    want = scene_ref.merge(tiles, 1, 0.2)
    assert want.shape[0] == 2
    assert torch.equal(res.rows.cpu(), torch.from_numpy(want))


@pytest.fixture(scope="module")
def model():
    from tests.modelgen import build_mirror
    return build_mirror("n", nc=15, seed=0, obj_bias=1.0, cls_bias=-1.0, det_gain=6.0).to(DEV)


def _composed(model, scene):
    """The reference chain from existing public calls: torch-built tiles -> model(tiles) -> non_max_suppression_obb ->
    rbox2poly -> scale_polys -> the CPU merge restatement."""
    from yolov5_obb_b200.general import non_max_suppression_obb
    origins = split_origins(*scene.shape[:2])
    tiles = _torch_tiles(scene, origins, 1024, 1056, 16).to(DEV)
    dets = non_max_suppression_obb(model(tiles)[0], 0.01, 0.4, multi_label=True, max_det=1500)
    rows = torch.zeros((len(origins), 1500, 7), device=DEV)
    counts = torch.tensor([d.shape[0] for d in dets], device=DEV)
    for t, d in enumerate(dets):
        rows[t, :d.shape[0]] = d
    tiles = [(l, u) + d for (l, u), d in zip(origins, _device_polys(rows, counts, 16.0))]
    return torch.from_numpy(scene_ref.merge(tiles, 15, 0.2)), int(counts.sum())


@pytest.mark.parametrize("batch", [4, 8])
def test_scene_detector_equals_composed_public_calls(model, batch):
    scene = _scene(1700, 2300, 2)
    want, n_tile_dets = _composed(model, scene)
    det = SceneDetector(model, batch_size=batch)
    got = det.det(scene.to(DEV)).rows.cpu()
    assert n_tile_dets > 1000 and want.shape[0] > 100
    assert torch.equal(got, want)
    assert torch.equal(det.det(scene.to(DEV)).rows.cpu(), got)


def test_refusals(model):
    det = SceneDetector(model, batch_size=2)
    scene = _scene(700, 900, 3)
    with pytest.raises(RuntimeError):
        det.det(scene)                                    # host tensor
    with pytest.raises(RuntimeError):
        det.det(scene.to(DEV).float())                    # not uint8
    with pytest.raises(RuntimeError):
        det.det(scene.to(DEV)[:, :, :2].contiguous())     # not [H, W, 3]
    with pytest.raises(RuntimeError):
        det.det(scene.to(DEV).permute(2, 0, 1))
    with pytest.raises(RuntimeError):
        SceneDetector(model, subsize=1024, gap=1024)
    with pytest.raises(RuntimeError, match="stride"):
        SceneDetector(types.SimpleNamespace(stride=torch.tensor([8.0, 16.0, 64.0])))   # 1056 is not a multiple of 64
    # one class with more candidates than the dense-mask bound
    T = 44
    rows = torch.zeros((T, 1500, 7), device=DEV)
    rows[..., 2:4] = 10.0
    rows[..., 5] = 0.5
    counts = torch.full((T,), 1500, dtype=torch.int64, device=DEV)
    org = torch.zeros((T, 2), dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match=str(_lib.SCENE_MAX_CLASS_CANDIDATES)):
        merge_tiles(rows, counts, org, 15)
