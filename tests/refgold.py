"""Results of the reference's own kernels, stored under tests/golden/ref_kernels.npz, so that the comparisons with the reference
run without it.

reference(key, compute, like=None) returns the stored result for `key`.  With the environment variable Y5OBB_RECORD_REF_GOLDEN
set to a file name, it instead calls compute() - which runs the reference kernels built into oracle/_ref by oracle/build_ref.py
- and writes every result it computed, together with the ones already stored, to that file when the process ends; that is how
ref_kernels.npz is made (`Y5OBB_RECORD_REF_GOLDEN=... python -m pytest tests/test_nms_gpu.py tests/test_oracle_nms.py
tests/test_poly_f32_gpu.py` on a GPU, then copy the file over tests/golden/ref_kernels.npz).

Arrays of more than LARGE elements are stored as a SHA-256 digest of their bytes and a sample of SAMPLE elements (every
(size // SAMPLE)-th): the caller passes its own result as `like`, which is returned when its digest equals the reference's; otherwise the call fails
and names the sampled elements that differ.  reference_sample(key, compute) returns the stored (flat indices, values) sample
for comparisons that allow a tolerance."""
import atexit
import hashlib
import os
from pathlib import Path

import numpy as np

GOLDEN = Path(__file__).resolve().parent / "golden" / "ref_kernels.npz"
LARGE = 100_000
SAMPLE = 32768
_stored = None
_recorded = {}
_keys = set()  # keys recorded in this process: what is stored under them is replaced


def _load():
    global _stored
    if _stored is None:
        _stored = dict(np.load(GOLDEN)) if GOLDEN.exists() else {}
    return _stored


def _digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _sample_idx(n: int) -> np.ndarray:
    return np.arange(0, n, max(1, n // SAMPLE))[:SAMPLE]


def _write(path):
    out = {k: v for k, v in _load().items() if not any(k == r or k.startswith(r + "/") for r in _keys)}
    out.update(_recorded)
    np.savez_compressed(path, **out)


def reference(key: str, compute, like=None) -> np.ndarray:
    rec_path = os.environ.get("Y5OBB_RECORD_REF_GOLDEN")
    if rec_path:
        ref = np.asarray(compute())
        if not _keys:
            atexit.register(_write, rec_path)
        _keys.add(key)
        for k in [k for k in _recorded if k == key or k.startswith(key + "/")]:
            del _recorded[k]
        if ref.size > LARGE:
            idx = _sample_idx(ref.size)
            _recorded[key + "/sha256"] = np.array(_digest(ref))
            _recorded[key + "/shape"] = np.array(ref.shape, np.int64)
            _recorded[key + "/sample"] = ref.ravel()[idx]
        else:
            _recorded[key] = ref
        return ref
    g = _load()
    if key in g:
        return g[key]
    assert key + "/sha256" in g, f"no stored reference result for {key!r} in {GOLDEN.name}"
    assert like is not None, f"{key!r} is stored as a digest: pass the result to compare as `like`"
    shape, sample = tuple(g[key + "/shape"]), g[key + "/sample"]
    idx = _sample_idx(int(np.prod(shape)))
    like = np.ascontiguousarray(np.asarray(like).astype(sample.dtype, copy=False))
    assert like.shape == shape, (key, like.shape, shape)
    if _digest(like) == str(g[key + "/sha256"]):
        return like
    got = like.ravel()[idx]
    bytes_of = lambda a: a.view(np.uint8).reshape(len(idx), -1)  # noqa: E731  (bitwise: NaN payloads and -0 count)
    bad = np.flatnonzero((bytes_of(got) != bytes_of(sample)).any(1))
    raise AssertionError(f"{key}: differs from the reference; {bad.size} of {len(idx)} sampled elements differ, "
                         f"first at flat indices {idx[bad[:5]]}: {got[bad[:5]]} vs {sample[bad[:5]]}")


def reference_sample(key: str, compute):
    """(flat indices, reference values) of the stored sample of a large result"""
    if os.environ.get("Y5OBB_RECORD_REF_GOLDEN"):
        reference(key, compute)
        return _sample_idx(int(np.prod(_recorded[key + "/shape"]))), _recorded[key + "/sample"]
    g = _load()
    assert key + "/sample" in g, f"no stored reference sample for {key!r} in {GOLDEN.name}"
    return _sample_idx(int(np.prod(g[key + "/shape"]))), g[key + "/sample"]
