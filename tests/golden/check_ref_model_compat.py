"""INTEGRATION.md B3, option 2 ("keep the reference Model object, replace _forward_once by InferenceEngine"): the engine
identifies modules by class NAME and reads a fixed set of attributes (engine.py).  This script - needs the reference checkout,
it imports the REFERENCE package (tests/golden/ref_import.py) - builds the reference's Model and the mirror from the same yaml and
checks that the engine's view of the two is identical, attribute by attribute, and that the reference's state_dict loads
into the mirror strictly (option 1).  It also stores what it compared - the reference's engine view, strides and parameter
names / shapes - as tests/golden/ref_model_view.json, which tests/test_ref_model_compat.py checks the mirror against.
Run as a script (the reference package puts top-level `models` / `utils` on sys.path and changes the working directory)."""
import json
import sys
from pathlib import Path

import torch

HERE = Path(__file__).resolve().parent
GOLDEN = HERE / "ref_model_view.json"
SIZES = ("n", "s", "m")


def conv_view(m):
    """what engine._conv_params / add_conv read of a Conv module"""
    c = m.conv
    return ("Conv", c.in_channels, c.out_channels, tuple(c.kernel_size), tuple(c.stride), tuple(c.padding), c.groups,
            c.bias is None, type(m.bn).__name__, float(m.bn.eps), type(m.act).__name__)


def engine_view(model):
    out = []
    for m in model.model:
        kind = type(m).__name__
        f = m.f if isinstance(m.f, int) else tuple(m.f)
        row = [kind, m.i, f]
        if kind == "Conv":
            row.append(conv_view(m))
        elif kind == "C3":
            row += [conv_view(m.cv1), conv_view(m.cv2), conv_view(m.cv3),
                    tuple((type(b).__name__, conv_view(b.cv1), conv_view(b.cv2), bool(b.add)) for b in m.m)]
        elif kind == "SPPF":
            k = getattr(m, "k", None)          # (the mirror keeps k, the reference the nn.MaxPool2d: engine.py reads either)
            if k is None:
                k = m.m.kernel_size if isinstance(m.m.kernel_size, int) else m.m.kernel_size[0]
                assert (m.m.stride, m.m.padding) == (1, k // 2)
            row += [conv_view(m.cv1), conv_view(m.cv2), k]
        elif kind == "Upsample":
            row += [m.scale_factor, m.mode]
        elif kind == "Concat":
            row.append(m.d)
        elif kind == "Detect":
            row += [m.nc, m.no, m.nl, m.na, tuple(m.anchors.shape), [round(float(s), 6) for s in m.stride],
                    [round(float(a), 5) for a in m.anchors.flatten()],
                    tuple((c.in_channels, c.out_channels, tuple(c.kernel_size)) for c in m.m)]
        else:
            raise SystemExit(f"module kind {kind} is not one the engine plans")
        out.append(tuple(row))
    return out


def record(model):
    """what is compared, in JSON form"""
    return json.loads(json.dumps({"view": engine_view(model), "stride": [round(float(s), 6) for s in model.stride],
                                  "params": [[n, list(p.shape)] for n, p in model.named_parameters()],
                                  "state_dict": sorted(model.state_dict().keys())}))


def main():
    sys.path.insert(0, str(HERE))
    import ref_import
    ref_import.setup()
    sys.path.insert(0, str(HERE.parents[1]))
    from models.yolo import Model as RefModel  # (the reference)
    from yolov5_obb_b200.yolo import Model as MirrorModel
    golden = {}
    for size in SIZES:
        torch.manual_seed(0)
        ref = RefModel(f"models/yolov5{size}.yaml", ch=3, nc=15)
        torch.manual_seed(0)
        mir = MirrorModel(f"yolov5{size}.yaml", ch=3, nc=15)
        a, b = engine_view(ref), engine_view(mir)
        assert len(a) == len(b), (len(a), len(b))
        for ra, rb in zip(a, b):
            assert ra == rb, f"yolov5{size}: the engine would see\n  reference {ra}\n  mirror    {rb}"
        assert [round(float(s), 6) for s in ref.stride] == [round(float(s), 6) for s in mir.stride]
        missing = mir.load_state_dict(ref.state_dict(), strict=True)
        assert not missing.missing_keys and not missing.unexpected_keys
        for (na, pa), (nb, pb) in zip(ref.named_parameters(), mir.named_parameters()):
            assert na == nb and pa.shape == pb.shape, (na, nb)
        golden[size] = record(ref)
        print(f"yolov5{size}: {len(a)} layers, {sum(p.numel() for p in ref.parameters())} parameters - identical engine view")
    GOLDEN.write_text(json.dumps(golden, separators=(",", ":")) + "\n")
    print("COMPAT OK")


if __name__ == "__main__":
    main()
