"""TEST INFRASTRUCTURE — stored outputs of the reference's marching-cubes CUDA operator
(``unbatched_mcube_forward_cuda``, oracle/build_ref_mcube.py), run through the reference wrapper's
per-view steps, kept in ``tests/golden/ref_cuda_mcube.npz`` in the format of oracle/ref_golden.py
(digest, scale, whole array or a fixed row sample), so that the tests need neither the reference's
sources nor a build of them.  A row is one vertex or one face.

Record on a GPU with oracle/_ref built by running tests/test_marching_cubes_gpu.py with
``KAOLIN_REF_CUDA_RECORD=1``; the file is rewritten when the process exits.
"""
import atexit
import hashlib
import os

import numpy as np

from . import ref_golden

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                    "ref_cuda_mcube.npz")
_recorded = {}
_stored = None


def _save():
    flat = {f"{c}.{n}.{f}": v for c, names in _recorded.items() for n, fields in names.items()
            for f, v in fields.items()}
    np.savez_compressed(PATH, **flat)


def _load():
    global _stored
    if _stored is None:
        _stored = {}
        if os.path.exists(PATH):
            with np.load(PATH) as z:
                for k in z.files:
                    c, name, field = k.rsplit(".", 2)
                    _stored.setdefault(c, {}).setdefault(name, {})[field] = z[k]
    return _stored


def _compact(case, name, t, full):
    """As ref_golden._compact, with a row being one row of the 2-D output (a vertex or a face), so
    that empty outputs can be stored too."""
    a = ref_golden._numpy(t)
    e = {"sha": np.array(ref_golden._digest(a)), "shape": np.array(a.shape, np.int64),
         "scale": np.array(np.abs(a.astype(np.float64)).max() if a.size else 0.0)}
    if full or a.shape[0] <= 2 * ref_golden.SAMPLE_ROWS:
        e["values"] = a
        return e
    rng = np.random.default_rng(int(hashlib.sha256(f"{case}.{name}".encode()).hexdigest()[:8], 16))
    e["rows"] = np.unique(rng.choice(a.shape[0], ref_golden.SAMPLE_ROWS, replace=False)).astype(np.int32)
    e["values"] = a[e["rows"]]
    return e


def rows(ref, name):
    """(row indices, values) stored for output ``name`` of a Reference."""
    e = ref._entry(name)
    return (e["rows"] if "rows" in e else np.arange(e["values"].shape[0])), e["values"]


def reference(case, live, names, full=()):
    """The reference operator's outputs ``names`` for ``case``; ``live()`` runs it (recording only).
    Outputs named in ``full`` are stored whole, the others as digest, scale and a row sample."""
    case = case.replace(".", "p")
    if ref_golden.RECORD:
        if not _recorded:
            atexit.register(_save)
        if case not in _recorded:
            out = live()
            _recorded[case] = {k: _compact(case, k, out[k], k in full) for k in names}
        return ref_golden.Reference(case, _recorded[case])
    stored = _load()
    if case not in stored:
        raise KeyError(f"no stored reference outputs for {case!r} in {PATH}")
    return ref_golden.Reference(case, stored[case])
