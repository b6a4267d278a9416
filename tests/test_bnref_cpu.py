"""CPU checks of tests/bnref.py: the launch geometry and addition-chain depth it restates from csrc/bn_train.cu, against a
replay of the kernels' exact fp32 summation order, and the rounding helpers its bounds are built from."""
import numpy as np
import pytest
import torch

from tests import bnref


def test_geometry_of_the_benchmarked_stem_layer():
    # 8 x 512 x 512 pixels, 48 channels on a 132-SM H100: 6 vector columns, 42 lanes, 528 blocks of 3972 pixels
    assert bnref.stat_layout(48) == (6, 6, 42)
    assert bnref.stat_geometry(8 * 512 * 512, 48, 132) == (528, 3972, 42)
    # per lane ceil(3972 / 42) = 95, 16-lane tree 2 + 15, reduce ceil(528 / 32) = 17 + 31
    assert bnref.stat_chain(8 * 512 * 512, 48, 132) == 95 + 2 + 15 + 17 + 31
    assert bnref.stat_layout(2056) == (257, 256, 1)       # the second column group
    assert bnref.stat_layout(8) == (1, 1, 256)
    assert bnref.stat_blocks(2, 48, 132) == 1
    # the element-wise kernels: 84 pixels per block step, capped at 8 blocks per SM; 2056 channels take two column groups
    assert bnref.colwise_grid(8 * 512 * 512, 48, 132) == (1056, 1)
    assert bnref.colwise_grid(85, 48, 132) == (2, 1)
    assert bnref.colwise_grid(3, 2056, 132) == (2, 2)


@pytest.mark.parametrize("npix,C,sms", [(2, 8, 4), (41, 48, 4), (42 * 16 * 16 + 1, 48, 4), (300, 16, 2), (255, 8, 1),
                                        (4100, 8, 2), (37, 2056, 3), (5000, 96, 3), (1, 128, 1)])
def test_chain_depth_and_bound_match_the_replayed_order(npix, C, sms):
    """The longest addition chain of the replayed kernel order equals stat_chain(), and the replayed fp32 sums lie within
    gamma(d) * sum|term| of the fp64 sums, at |mean| / sigma = 0 and 100."""
    rng = np.random.default_rng(npix + C)
    for ratio in (0, 100):
        x = (rng.standard_normal((npix, C)) + ratio).astype(np.float32)
        x = torch.from_numpy(x).bfloat16().float().numpy()
        s, q, depth = bnref.emulate_stats(x, sms)
        d = bnref.stat_chain(npix, C, sms)
        assert depth == d
        xd = x.astype(np.float64)
        assert np.all(np.abs(s - xd.sum(0)) <= bnref.gamma(d) * np.abs(xd).sum(0))
        assert np.all(np.abs(q - (xd * xd).sum(0)) <= bnref.gamma(d) * (xd * xd).sum(0))


def test_rounding_helpers():
    assert bnref.half_ulp_bf16(torch.tensor([1.0])).item() == 2.0 ** -8
    assert bnref.half_ulp_bf16(torch.tensor([1.5])).item() == 2.0 ** -8
    assert bnref.half_ulp_bf16(torch.tensor([2.0])).item() == 2.0 ** -7
    assert bnref.ulp32(torch.tensor([1.0])).item() == 2.0 ** -23
    assert bnref.ulp32(torch.tensor([0.75])).item() == 2.0 ** -24
    # one round-to-nearest into bf16 of an fp32 value errs by at most half_ulp_bf16 of the value
    x = torch.randn(100000, generator=torch.Generator().manual_seed(0)) * 1e3
    assert ((x.bfloat16().double() - x.double()).abs() <= bnref.half_ulp_bf16(x)).all()
    assert bnref.gamma(100) > 100 * 2.0 ** -24


def test_routing_references():
    g = torch.Generator().manual_seed(1)
    g2 = torch.randint(-20, 21, (2, 6, 8, 16), generator=g).bfloat16()     # integers: every order sums exactly
    old = torch.randint(-20, 21, (2, 3, 4, 16), generator=g).bfloat16()
    want = g2.float().view(2, 3, 2, 4, 2, 16).sum((2, 4))
    assert torch.equal(bnref.upsample2x_bwd_ref(g2), want.bfloat16())
    assert torch.equal(bnref.upsample2x_bwd_ref(g2, old), (want + old.float()).bfloat16())
    # max-pool routing: ties go to the first maximum in row-major window order, the gradient is conserved
    x = torch.zeros(1, 3, 3, 1).bfloat16()
    r = bnref.maxpool5_route(x, torch.ones(1, 3, 3, 1))
    assert r[0, 0, 0, 0].item() == 9 and r.sum().item() == 9
    gd = torch.randn(2, 3, 2, 2, 5, generator=g)
    out = bnref.detect_grad_pack_ref(gd, 8)
    assert out.shape == (2, 2, 2, 24)
    assert torch.equal(out.view(2, 2, 2, 3, 8)[..., 5:], torch.zeros(2, 2, 2, 3, 3, dtype=torch.bfloat16))
    assert torch.equal(out.view(2, 2, 2, 3, 8)[..., :5], gd.permute(0, 2, 3, 1, 4).bfloat16())

