"""Import the REFERENCE python package from the reference checkout (oracle/build_ref.REF) with the
environment shims SURVEY §8(c) lists: stub matplotlib/seaborn, cwd at the reference root (Arial.ttf),
numpy.int alias, and the reference's nms_rotated_ext provided by oracle/_ref (its own CPU kernel).
Used only by the make_*_golden.py scripts."""
import os
import sys
import tempfile
import types
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
from oracle.build_ref import REF  # noqa: E402


def setup():
    assert REF.exists(), f"the reference checkout {REF} is missing"
    stubs = Path(tempfile.mkdtemp(prefix="refstubs_"))
    (stubs / "matplotlib").mkdir()
    (stubs / "matplotlib" / "__init__.py").write_text(
        "def use(*a, **k): pass\ndef rc(*a, **k): pass\nclass _C:\n    def __getattr__(self, k): return lambda *a, **kw: None\ncolors = _C()\n")
    (stubs / "matplotlib" / "pyplot.py").write_text("def __getattr__(k):\n    return lambda *a, **kw: None\n")
    (stubs / "seaborn.py").write_text("def __getattr__(k):\n    return lambda *a, **kw: None\n")
    sys.path.insert(0, str(stubs))
    sys.path.insert(0, str(ROOT))
    sys.path.insert(0, str(REF))
    os.chdir(REF)
    import numpy as np
    if not hasattr(np, "int"):
        np.int = int
    os.environ.setdefault("TORCH_FORCE_NO_WEIGHTS_ONLY_LOAD", "1")
    # the reference's compiled extension: its own CPU kernel, built by oracle/build_ref.py
    from oracle.build_ref import build, load_ref
    build()
    ref = load_ref()
    ext = types.ModuleType("utils.nms_rotated.nms_rotated_ext")
    ext.nms_rotated = lambda d, s, t: ref.nms_rotated_cpu(d, s, float(t))
    ext.nms_poly = lambda *a, **k: (_ for _ in ()).throw(RuntimeError("nms_poly unbuildable (THC)"))
    sys.modules["utils.nms_rotated.nms_rotated_ext"] = ext
