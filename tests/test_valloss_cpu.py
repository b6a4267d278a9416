"""CPU tests of the validation loss (val.py:198-199): the fp32 oracle path (the mirror model through oracle/model_ref.forward,
then oracle/loss_ref.compute_loss on its raw Detect outputs) against the REFERENCE model and ComputeLoss
(tests/golden/valloss_golden.npz, made by make_valloss_golden.py), and the golden's val.py accumulation."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import loss_ref, model_ref
from tests import vallossgen as VG
from tests.modelgen import build_mirror

ROOT = Path(__file__).resolve().parents[1]
G = np.load(ROOT / "tests" / "golden" / "valloss_golden.npz")


def oracle_items(m, emulate_bf16=False):
    """Per batch, loss_ref.compute_loss on the oracle's raw Detect outputs: [N_BATCHES, 4] fp32."""
    det = m.model[-1]
    hyp = loss_ref.scaled_hyp(loss_ref.DEFAULT_HYP, 3, 15, VG.HYP_IMGSZ)
    out = []
    for i in range(VG.N_BATCHES):
        im, tg = VG.batch(i)
        assert im.long().sum().item() == int(G[f"batch{i}/im_sum"])
        assert np.array_equal(tg.numpy(), G[f"batch{i}/targets"])
        _, raw = model_ref.forward(m, im.float() / 255, emulate_bf16=emulate_bf16)
        out.append(loss_ref.compute_loss(raw, tg, det.anchors, det.stride, hyp, 15)[1].numpy())
    return np.stack(out)


def test_hyp_is_the_scaled_finetune_hyp():
    h = loss_ref.scaled_hyp(loss_ref.DEFAULT_HYP, 3, 15, VG.HYP_IMGSZ)
    np.testing.assert_allclose(G["hyp"], [h["box"], h["obj"], h["cls"], h["theta"], h["anchor_t"]], rtol=1e-12)


@pytest.mark.parametrize("size", VG.SIZES)
def test_oracle_items_match_reference(size):
    got = oracle_items(build_mirror(size, nc=15, seed=0, obj_bias=VG.OBJ_BIAS))
    want = G[f"{size}/items"]
    assert np.all(want > 0)
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=0)


@pytest.mark.parametrize("size", VG.SIZES)
def test_golden_accumulation_is_val_py_333(size):
    """val.py:179 / 199 / 333: an fp32 sum of the per-batch items in batch order, then the CPU division by the batch count."""
    acc = torch.zeros(4)
    for it in G[f"{size}/items"]:
        acc += torch.from_numpy(it)
    assert (acc / VG.N_BATCHES).tolist() == G[f"{size}/results"].tolist()
