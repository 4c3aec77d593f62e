"""TEST INFRASTRUCTURE — stored outputs of the reference's spherical-Gaussian CUDA operator
(oracle/build_ref_sg.py), kept in ``tests/golden/ref_cuda_sg.npz`` in the format of
oracle/ref_golden.py (digest, scale, whole array or a fixed row sample), so that the GPU tests need
neither the reference's sources nor a build of them.  The mesh operators' file, tests/golden/ref_cuda.npz,
is a separate store and is not touched.

Record on a GPU with oracle/_ref built by running the GPU tests with ``KAOLIN_REF_CUDA_RECORD=1``.
"""
import atexit
import os

import numpy as np

from . import ref_golden

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ref_cuda_sg.npz")
_recorded = {}


def _save():
    flat = {f"{c}.{n}.{f}": v for c, names in _recorded.items() for n, fields in names.items()
            for f, v in fields.items()}
    np.savez_compressed(PATH, **flat)


def reference(case, live, names):
    """The reference operator's outputs ``names`` for ``case``; ``live()`` runs it (recording only)."""
    if ref_golden.RECORD:
        if not _recorded:
            atexit.register(_save)
        out = live()
        _recorded[case] = {k: ref_golden._compact(case, k, out[k], False) for k in names}
        return ref_golden.Reference(case, _recorded[case])
    if not os.path.exists(PATH):
        raise KeyError(f"no stored reference outputs in {PATH}")
    stored = {}
    with np.load(PATH) as z:
        for k in z.files:
            c, name, field = k.rsplit(".", 2)
            if c == case:
                stored.setdefault(name, {})[field] = z[k]
    if not stored:
        raise KeyError(f"no stored reference outputs for {case!r} in {PATH}")
    return ref_golden.Reference(case, stored)
