"""The CPU restatement of the validation metrics (oracle/valmetrics_ref.py) against the reference's own ap_per_class, fitness
and val.py tail (tests/golden/valmetrics_golden.npz), bit for bit, and its stats accumulation against the per-image stats
val.py:209-250 built from the valgen batches."""
from pathlib import Path

import numpy as np
import pytest

from oracle import valmetrics_ref as V
from tests.valmetricsgen import val_batches

G = np.load(Path(__file__).resolve().parent / "golden" / "valmetrics_golden.npz")
CASES = [("mixed10", 8), ("mixed1", 8), ("notp", 8), ("small", 8), ("valgen", 15)]


def case_stats(name):
    pre = "valgen/stats" if name == "valgen" else f"{name}/in"
    return [G[f"{pre}/{k}"] for k in ("tp", "conf", "pred_cls", "target_cls")]


def assert_equals_golden(name, got):
    assert np.array_equal(np.array(got["results"], np.float64), G[f"{name}/results"])
    assert np.array_equal(got["maps"], G[f"{name}/maps"])
    assert np.array_equal(V.fitness(np.array(got["results"]).reshape(1, -1)), G[f"{name}/fitness"])
    if f"{name}/ap_full" not in G:   # the stats[0].any() gate: nothing else is computed
        assert got["ap_class"].size == 0
        return
    c = got["curves"]
    for k in ("tp", "fp", "p", "r", "f1", "ap_class", "p_curve", "r_curve"):
        assert np.array_equal(c[k], G[f"{name}/{k}"]), k
    assert np.array_equal(c["ap"], G[f"{name}/ap_full"])
    assert np.array_equal(got["ap50"], G[f"{name}/ap50"]) and np.array_equal(got["ap"], G[f"{name}/ap"])


@pytest.mark.parametrize("name,nc", CASES)
def test_restatement_equals_reference(name, nc):
    assert_equals_golden(name, V.val_metrics(case_stats(name), nc))


def test_cases_cover_the_edges():
    tp, conf, cls, tcls = case_stats("mixed10")
    assert tp.shape[1] == 10 and case_stats("mixed1")[0].shape[1] == 1
    assert set(np.unique(cls)) - set(np.unique(tcls)) == {2.0}          # predictions of a class without labels
    assert set(np.unique(tcls)) - set(np.unique(cls)) == {1.0}          # labels without predictions
    assert (cls == 3).sum() == 1 and tp[cls == 4].all()                 # one prediction; an all-TP class
    assert not case_stats("notp")[0].any()


def test_accumulation_equals_val_loop():
    """image_stats on the valgen batches reproduces the per-image entries of val.py:209-250: images with detections and
    no labels (all-False rows), images with labels and no detections (empty rows, their labels)."""
    per_image, lengths, tl = G["valgen/per_image"], G["valgen/lengths"], G["valgen/tcls_lengths"]
    tp = G["valgen/stats/tp"]
    offs = np.concatenate([[0], np.cumsum(lengths)])
    stats = []
    for bi, (dets, counts, targets, _) in enumerate(val_batches()):
        correct = np.zeros((dets.shape[0], dets.shape[1], 10), bool)
        for e, (b, si) in enumerate(per_image.tolist()):
            if b == bi:
                correct[si, :lengths[e]] = tp[offs[e]:offs[e + 1]]
        stats += V.image_stats(correct, dets, counts, targets, 10)
    assert [len(s[1]) for s in stats] == lengths.tolist() and [len(s[3]) for s in stats] == tl.tolist()
    assert 0 in lengths.tolist() and 0 in tl.tolist()
    cat = V.concat_stats(stats)
    for got, k in zip(cat, ("tp", "conf", "pred_cls", "target_cls")):
        want = G[f"valgen/stats/{k}"]
        assert got.dtype == want.dtype and np.array_equal(got, want), k
