"""train.py --freeze without a GPU: which parameters TrainStep's freeze rule freezes, and which gradients the backward plan's
liveness rule keeps (layout.grad_liveness), on the mirror Model."""
import pytest

from yolov5_obb_b200 import yolo as Y
from yolov5_obb_b200.layout import grad_liveness, shapes, sources
from yolov5_obb_b200.train_step import TrainStep, freeze_layers

CASES = [[10], [0, 1, 2], [24], [0], [5, 7], [0, 99], [40]]


def _expected_frozen(model, freeze):
    """train.py:126-131 restated by layer index: [n] is layers 0..n-1, a longer list the layers it names; a parameter is
    frozen when its module path starts with one of those layers."""
    layers = set(freeze) if len(freeze) > 1 else set(range(freeze[0]))
    return {n for n, _ in model.named_parameters() if n.split(".")[0] == "model" and int(n.split(".")[1]) in layers}


def _reachable(mods, owns):
    """Nodes reachable from a node that owns a trainable parameter along the forward edges (a search from the sources of
    the gradient, independent of layout.needs_grad's single pass in layer order)."""
    consumers = {m.i: [] for m in mods}
    for m in mods:
        if m.i:
            for s in sources(m):
                consumers[s].append(m.i)
    seen, todo = set(), [m.i for m in mods if owns(m)]
    while todo:
        i = todo.pop()
        if i not in seen:
            seen.add(i)
            todo += consumers[i]
    return seen


def _trainable(m):
    return any(p.requires_grad for p in m.parameters())


@pytest.mark.parametrize("cfg", ["n", "s", "m", "s6"])
@pytest.mark.parametrize("freeze", CASES)
def test_freeze_rule_matches_train_py(cfg, freeze):
    m = Y.Model(f"yolov5{cfg}.yaml", nc=15)
    for p in list(m.parameters())[::7]:     # the rule sets every flag: what was set before does not matter
        p.requires_grad_(False)
    frozen = freeze_layers(m, freeze)
    want = _expected_frozen(m, freeze)
    assert set(frozen) == want
    assert {n for n, p in m.named_parameters() if not p.requires_grad} == want
    if freeze == [0]:
        assert not want
    if freeze == [0, 99]:   # index 99 names no layer: only layer 0 is frozen
        assert want and all(n.startswith("model.0.") for n in want)


@pytest.mark.parametrize("cfg", ["n", "s", "m", "s6"])
@pytest.mark.parametrize("freeze", CASES)
def test_liveness_rule(cfg, freeze):
    m = Y.Model(f"yolov5{cfg}.yaml", nc=15)
    freeze_layers(m, freeze)
    mods = list(m.model)
    ch, _ = shapes(mods, 256, 256)
    need, windows = grad_liveness(mods, ch, _trainable)
    assert need == _reachable(mods, _trainable)
    for m_ in mods:
        if type(m_).__name__ != "Concat":
            continue
        if m_.i not in need:
            assert m_.i not in windows
            continue
        off, live = 0, []
        for s in sources(m_):
            if s in need:
                live.append((off, off + ch[s]))
            off += ch[s]
        assert sum(b - a for a, b in windows[m_.i]) == sum(b - a for a, b in live)
        assert all(any(a <= lo and hi <= b for a, b in windows[m_.i]) for lo, hi in live)


def test_liveness_yolov5s_backbone_frozen():
    """--freeze 10 on yolov5s: gradients of layers 10-24 only; Concat 12 = [up(10), 6] and 16 = [up(14), 4] need only the
    channels of their head-path input, [0, C)."""
    m = Y.Model("yolov5s.yaml", nc=15)
    freeze_layers(m, [10])
    mods = list(m.model)
    ch, _ = shapes(mods, 256, 256)
    need, windows = grad_liveness(mods, ch, _trainable)
    assert need == set(range(10, 25))
    assert windows[12] == [(0, ch[11])] and ch[11] < ch[12]
    assert windows[16] == [(0, ch[15])] and ch[15] < ch[16]
    assert windows[19] == [(0, ch[19])] and windows[22] == [(0, ch[22])]


@pytest.mark.parametrize("freeze,want", [([0], set(range(25))), ([0, 1, 2], set(range(3, 25))), ([24], {24}),
                                         ([5, 7], set(range(25))), ([11], set(range(13, 25)))])
def test_liveness_yolov5s_cases(freeze, want):
    m = Y.Model("yolov5s.yaml", nc=15)
    freeze_layers(m, freeze)
    mods = list(m.model)
    ch, _ = shapes(mods, 256, 256)
    need, windows = grad_liveness(mods, ch, _trainable)
    assert need == want
    if freeze == [11]:   # layers 0-10 frozen: Concat 12 needs no gradient, Concat 22 = [21, 10] only its first input's
        assert 12 not in windows and windows[16] == [(0, ch[15])] and windows[22] == [(0, ch[21])]


def test_freezing_everything_is_refused():
    m = Y.Model("yolov5n.yaml", nc=15).train()
    with pytest.raises(RuntimeError, match="nothing is left to train"):
        TrainStep(m, batch_size=16, imgsz=256, freeze=[25])
