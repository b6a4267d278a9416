"""The model walk both plans share (yolov5_obb_b200/layout.py) on the CPU: every layer's shape against the fp32 oracle's own
forward, the Concat routing against the oracle's Concat outputs, the stem weight rewrite and its gradient inverse, and the
graphs the routing refuses."""
import pytest
import torch

from oracle import model_ref
from tests.modelgen import build_mirror
from yolov5_obb_b200.layout import _is, route, shapes, sources, stem_grad, stem_weight


def _bf16_new(B):
    return lambda h, w, c: torch.zeros((B, h, w, c), dtype=torch.bfloat16)


@pytest.mark.parametrize("size,H,W", [("s", 192, 320), ("s6", 256, 384)])
def test_shapes_and_routing_match_the_oracle(size, H, W):
    m = build_mirror(size, nc=15, seed=0)
    layers = list(m.model)
    B = 2
    x = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(1))
    _, ys = model_ref.forward(m, x, return_layers=True)
    ch, hw = shapes(layers, H, W)
    for mm, y in zip(layers[:-1], ys):
        assert (ch[mm.i],) + hw[mm.i] == tuple(y.shape[1:]), f"layer {mm.i} ({type(mm).__name__})"

    out, up_of = route(layers, ch, hw, _bf16_new(B))
    for i, src in up_of.items():
        assert _is(layers[i], "Conv") and any(_is(mm, "Upsample") and sources(mm) == [i] and out[mm.i] is src
                                              for mm in layers)
    # every layer output written where the routing put it: each Concat buffer then holds the oracle's Concat output
    for mm in layers[:-1]:
        if not _is(mm, "Concat"):
            out[mm.i].view().copy_(ys[mm.i].permute(0, 2, 3, 1))
    n_cat = 0
    for mm in layers[:-1]:
        if _is(mm, "Concat"):
            off = 0
            for s in sources(mm):
                assert out[s].buf is out[mm.i].buf and out[s].c_off == off and out[s].C == ch[s], f"Concat {mm.i} input {s}"
                off += ch[s]
            assert off == out[mm.i].C == out[mm.i].buf.shape[3]
            want = ys[mm.i].permute(0, 2, 3, 1).bfloat16()
            assert torch.equal(out[mm.i].view(), want), f"Concat {mm.i}"
            n_cat += 1
    assert n_cat == (4 if size == "s" else 6)


def test_stem_gradient_inverse():
    w = torch.randn(32, 3, 6, 6, generator=torch.Generator().manual_seed(2))
    w3 = stem_weight(w)                                    # [Cout, 48, 3 (ty), 1]
    assert w3.shape == (32, 48, 3, 1)
    assert not w3.view(32, 3, 16, 3)[:, :, 12:].any()      # channels 12-15 of every window are padding
    dw = w3[..., 0].permute(2, 0, 1).contiguous()          # the stem wgrad's layout [ty][Cout][48]
    g = torch.full_like(w, float("nan"))
    stem_grad(dw.view(-1), g)
    assert torch.equal(g, w)


def test_route_refuses_a_layer_feeding_two_concats():
    m = build_mirror("s")
    layers = list(m.model)
    # yolov5s: Concat 12 joins [11, 6] and Concat 19 joins [18, 14], all at stride 16; let 19 read layer 6 as well
    assert _is(layers[19], "Concat") and sources(layers[19]) == [18, 14] and 6 in sources(layers[12])
    layers[19].f = [-1, 6]
    ch, hw = shapes(layers, 256, 256)
    with pytest.raises(RuntimeError, match="two Concats"):
        route(layers, ch, hw, _bf16_new(1))
