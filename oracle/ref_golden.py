"""TEST INFRASTRUCTURE — stored outputs of the reference's own CUDA kernels (oracle/_ref).

The GPU tests that compare with the reference's kernels read ``tests/golden/ref_cuda.npz``, so
they need neither the reference's sources nor a build of them.  For every case and output the file
keeps a SHA-256 digest of the whole array (bit-exact comparisons), its largest magnitude (the scale
of max-normalised gradient errors) and a fixed sample of its rows: a row is a pixel of an image
output or a face of a gradient output; half of the sample is drawn from the rows that carry a value
(covered pixels, faces with a gradient), half from all rows, plus the row of the largest magnitude.
Outputs named in ``full=``, and outputs of at most 2 * SAMPLE_ROWS rows, are stored whole.

A test may keep its cases in a store file of its own (``path=``), with fewer sampled rows
(``sample_rows=``) and, for outputs it only compares bit for bit (``digest_only=``), nothing but the
digest and the shape: the float32 binning matrix keeps thousands of outputs in
``tests/golden/ref_cuda_binning.npz`` that way.

Regenerate on a GPU with oracle/_ref built (``oracle/build_ref.py``) by running the GPU tests with
``KAOLIN_REF_CUDA_RECORD=1``: every ``reference()`` call then runs the reference and each store it
recorded into is rewritten when the process exits.
"""
import atexit
import hashlib
import os

import numpy as np
import torch

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ref_cuda.npz")
RECORD = os.environ.get("KAOLIN_REF_CUDA_RECORD") == "1"
SAMPLE_ROWS = 256         # outputs of at most 2 * SAMPLE_ROWS rows are stored whole
_PIXEL_DIMS = 3          # (B, H, W[, D]) image outputs; everything else is (B, F, ...) per face

_stored = {}       # path -> {case: {name: {field: array}}}
_recorded = {}     # path -> {case: ...}, the cases recorded by this process


def _numpy(t):
    if isinstance(t, np.ndarray):
        return np.ascontiguousarray(t)
    t = t.detach().contiguous()
    if t.dtype == torch.bfloat16:
        t = t.view(torch.int16)
    return t.cpu().numpy()


def _digest(a):
    return hashlib.sha256(str(a.dtype).encode() + str(a.shape).encode() + a.tobytes()).hexdigest()


def _row_view(name, a):
    lead = _PIXEL_DIMS if name in ("face_idx", "soft_mask", "features", "features_bf16", "weights") else 2
    return a.reshape(int(np.prod(a.shape[:lead])), -1)


def _compact(case, name, t, full, sample_rows=SAMPLE_ROWS, digest_only=False):
    a = _numpy(t)
    e = {"sha": np.array(_digest(a)), "shape": np.array(a.shape, np.int64)}
    if digest_only:
        return e
    rows = _row_view(name, a)
    mag = np.abs(rows.astype(np.float64))
    e["scale"] = np.array(mag.max() if mag.size else 0.0)
    if full or rows.shape[0] <= 2 * sample_rows:
        e["values"] = rows
        return e
    rng = np.random.default_rng(int(hashlib.sha256(f"{case}.{name}".encode()).hexdigest()[:8], 16))
    marked = np.flatnonzero((rows != -1).any(1) if name == "face_idx" else (rows != 0).any(1))
    n = min(sample_rows // 2, marked.size)
    pick = [marked[rng.choice(marked.size, n, replace=False)] if n else np.zeros(0, np.int64),
            rng.choice(rows.shape[0], sample_rows // 2, replace=False)]
    if mag.size:
        pick.append(np.array([np.unravel_index(np.argmax(mag), mag.shape)[0]]))
    e["rows"] = np.unique(np.concatenate(pick)).astype(np.int32)
    e["values"] = rows[e["rows"]]
    return e


class Reference:
    """The stored outputs of one case."""

    def __init__(self, case, entries, path=PATH):
        self.case, self.e, self.path = case, entries, path

    def _entry(self, name):
        if name not in self.e:
            raise KeyError(f"{self.case}: no stored reference output {name!r} in {self.path}")
        return self.e[name]

    def equal(self, name, ours):
        """Bit-exact: same dtype, shape and bytes as the reference's whole output."""
        return _digest(_numpy(ours)) == str(self._entry(name)["sha"])

    def scale(self, name):
        return float(self._entry(name)["scale"])

    def rows(self, name):
        e = self._entry(name)
        return e["rows"] if "rows" in e else np.arange(len(e["values"]))

    def pair(self, name, ours):
        """(ours, reference) on the stored rows, as numpy arrays of the reference's row layout."""
        e = self._entry(name)
        a = _numpy(ours)
        assert tuple(a.shape) == tuple(e["shape"]), (self.case, name, a.shape, tuple(e["shape"]))
        return _row_view(name, a)[self.rows(name)], e["values"]


def _load(path):
    if path not in _stored:
        _stored[path] = {}
        if os.path.exists(path):
            with np.load(path) as z:
                for k in z.files:
                    case, name, field = k.rsplit(".", 2)
                    _stored[path].setdefault(case, {}).setdefault(name, {})[field] = z[k]
    return _stored[path]


def _save():
    for path, recorded in _recorded.items():
        merged = {c: dict(v) for c, v in _load(path).items()}
        merged.update(recorded)
        flat = {f"{c}.{n}.{f}": v for c, names in merged.items() for n, fields in names.items()
                for f, v in fields.items()}
        np.savez_compressed(path, **flat)


def reference(case, live, names=("face_idx", "features", "soft_mask", "grad_fvi", "grad_ff"), full=(),
              path=PATH, sample_rows=SAMPLE_ROWS, digest_only=()):
    """The reference's outputs ``names`` for ``case`` in the store ``path``.  ``live()`` runs the
    reference (oracle/_ref) and returns {name: tensor}; it is called only when recording.  Outputs in
    ``full`` are stored whole, those in ``digest_only`` as their digest and shape alone, the others
    whole up to 2 * sample_rows rows and as a sample of sample_rows rows above that."""
    case = case.replace(".", "p")
    if RECORD:
        if not _recorded:
            atexit.register(_save)
        out = {k: v for k, v in live().items() if k in names}
        entries = {k: _compact(case, k, v, k in full, sample_rows, k in digest_only) for k, v in out.items()}
        _recorded.setdefault(path, {})[case] = entries
        return Reference(case, entries, path)
    stored = _load(path)
    if case not in stored:
        raise KeyError(f"no stored reference outputs for {case!r} in {path}")
    return Reference(case, stored[case], path)
