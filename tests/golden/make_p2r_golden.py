"""Golden vectors for poly2rbox from the REFERENCE's utils/rboxs_utils.py:39-81 (whose arithmetic is cv2.minAreaRect,
opencv-python 4.13.0 when they were made; requirements.txt:6 only gives a lower bound >= 4.5.4).
python tests/golden/make_p2r_golden.py"""
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import ref_import  # noqa: E402

ref_import.setup()
sys.path.insert(0, str(HERE.parents[1]))
from utils.rboxs_utils import poly2rbox  # noqa: E402
from tests.p2rgen import p2r_polys  # noqa: E402


def main():
    import cv2
    P = p2r_polys(seed=0)
    out = {"polys": P, "rbox_pi": poly2rbox(P, use_pi=True), "rbox_deg": poly2rbox(P, use_pi=False),
           "cv2_version": np.array(cv2.__version__)}
    rb, csl = poly2rbox(P[:64], num_cls_thata=180, radius=2.0, use_pi=True, use_gaussian=True)
    out["csl_rbox"] = rb
    out["csl"] = csl.astype(np.float32)
    np.savez_compressed(HERE / "p2r_golden.npz", **out)
    print({k: getattr(v, "shape", v) for k, v in out.items()})


if __name__ == "__main__":
    main()
