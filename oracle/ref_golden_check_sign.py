"""TEST INFRASTRUCTURE — stored outputs of the reference's point-in-mesh CUDA operator
(``unbatched_mesh_intersection_cuda``, oracle/build_ref_check_sign.py), kept in
``tests/golden/ref_cuda_check_sign.npz`` in the format of oracle/ref_golden.py (digest, scale, whole
array or a fixed row sample), so that the tests need neither the reference's sources nor a build of
them.  A row is one (view, point) count.

Record on a GPU with oracle/_ref built by running tests/test_check_sign_gpu.py with
``KAOLIN_REF_CUDA_RECORD=1``; the file is rewritten when the process exits.
"""
import atexit
import os

import numpy as np

from . import ref_golden

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                    "ref_cuda_check_sign.npz")
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


def reference(case, live, names, full=()):
    """The reference operator's outputs ``names`` for ``case``; ``live()`` runs it (recording only).
    Outputs named in ``full`` are stored whole, the others as digest, scale and a row sample."""
    case = case.replace(".", "p")
    if ref_golden.RECORD:
        if not _recorded:
            atexit.register(_save)
        if case not in _recorded:
            out = live()
            _recorded[case] = {k: ref_golden._compact(case, k, out[k], k in full) for k in names}
        return ref_golden.Reference(case, _recorded[case])
    stored = _load()
    if case not in stored:
        raise KeyError(f"no stored reference outputs for {case!r} in {PATH}")
    return ref_golden.Reference(case, stored[case])
