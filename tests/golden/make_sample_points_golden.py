"""Regenerate tests/golden/sample_points.npz from the reference's own face_areas, packed_face_areas,
sample_points and packed_sample_points, run on the CPU through oracle/ref_import.py (needs the reference
sources).

The reference draws its randomness from ``Categorical.sample`` and two ``torch.rand`` calls.  Both are
patched to return what the random-stream contract of kaolin_b200 (oracle/sample_points.py) gives for
the scene's fixed key: the face choices and the uniforms u_raw and v.  The reference then does
everything else itself: the gathers, the interpolation with its rounding and, through CPU autograd, the
gradients for fixed upstream gradients.  torch's CPU sqrt is not correctly rounded (with AVX-512 it
differs from IEEE sqrt in about 0.7 % of float32 and float64 inputs); the reference's CUDA path and
this library use the correctly rounded sqrt, so the maker runs the reference with ``torch.sqrt``
replaced by numpy's, whose backward is torch's (grad / (2 * result)).  On the CPU the reference's
tile_to_packed takes its torch path, so the packed forms need no stand-in for its CUDA operator.

The maker asserts that the oracle's areas, points and features equal the reference's bit for bit, and
that no stored sample's t = r * c_last lies within 4 * F * 2^-53 * c_last of a CDF boundary, so that no
summation order of the CDF can change a stored choice.

    python tests/golden/make_sample_points_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from kaolin_b200 import synthetic  # noqa: E402
from oracle import ref_import  # noqa: E402
from oracle import sample_points as osp  # noqa: E402

OUT = os.path.join(HERE, "sample_points.npz")
DTYPES = {"f32": np.float32, "f64": np.float64}
INDICES = ("faces", "choices", "first_idx", "num_faces")   # stored as int32; the tests read them as int64


def _ico(level, rng, jitter, scale=1.0):
    v, f = synthetic.icosphere(level)
    v = np.asarray(v, np.float64) * scale
    v = v + rng.normal(scale=jitter, size=v.shape)
    return np.round(v * 1024) / 1024, np.asarray(f, np.int64)     # on a 2^-10 grid: a small fixture


def scenes():
    """name -> dict(vertices (B, V, 3) float64, faces, N, key, areas, D); packed scenes have first_idx
    and num_faces instead of a batch dimension."""
    rng = np.random.default_rng(7)
    s = {}
    v0, f = _ico(3, rng, 0.02)
    v1, _ = _ico(3, rng, 0.02, 1.3)
    s["ico3"] = dict(vertices=np.stack([v0, v1]), faces=f, N=400, key=0x1234_5678_9ABC_DEF0, D=3)
    # zero-area faces (a repeated vertex, collinear vertices) and duplicate faces
    dv = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 0, 0], [0, 0, 1], [1, 1, 1]], np.float64)
    df = np.array([[0, 1, 2], [0, 0, 2], [0, 1, 3], [1, 2, 4], [1, 2, 4], [2, 4, 5], [3, 3, 3], [0, 1, 2]], np.int64)
    s["degenerate"] = dict(vertices=dv[None], faces=df, N=300, key=-0x0123_4567_89AB_CDEF, D=2)
    # areas from about 1e-7 to 1: triangle k scaled by 10^(-k/2)
    sv, sf = [], []
    for k in range(15):
        a = 10.0 ** (-k / 2.0)
        sv += [[3 * k, 0, 0], [3 * k + 2 * a, 0, 0], [3 * k, a, 0.5 * a]]
        sf.append([3 * k, 3 * k + 1, 3 * k + 2])
    sv = np.array(sv, np.float64)
    s["spread"] = dict(vertices=np.stack([sv, sv * 1.5]), faces=np.array(sf, np.int64), N=400, key=42, D=0)
    s["single"] = dict(vertices=np.array([[[0.5, -1, 2], [1.5, 0.25, 2], [0, 1, -1]]], np.float64),
                       faces=np.array([[0, 1, 2]], np.int64), N=64, key=-1, D=3)
    gv, gf = _ico(2, rng, 0.03)
    areas = np.round(rng.uniform(0.0, 5.0, size=(2, gf.shape[0])) * 64) / 64
    areas[:, ::3] = 0.0
    s["given_areas"] = dict(vertices=np.stack([gv, gv * 0.5]), faces=gf, N=300, key=0x7FFF_FFFF_FFFF_FFFF,
                            areas=areas, D=0)
    # the reference's packed test scene (test_trianglemesh.py:247-266)
    s["packed_ref"] = dict(vertices=np.array([[0., 0., 0.], [0., 0., 1.], [0., 1., 0.], [2., 0., 0.2],
                                              [0., 0., 0.], [0., 1., 1.], [2., 0., 0.]]),
                           first_idx=np.array([0, 4, 7], np.int64), faces=np.array([[0, 1, 2], [1, 0, 3], [0, 1, 2]]),
                           num_faces=np.array([2, 1], np.int64), N=200, key=99, packed=True)
    pv, pf, first, nfm = [], [], [0], []
    for level, scale in ((1, 1.0), (2, 0.7), (0, 2.0)):
        v, f = _ico(level, rng, 0.01, scale)
        pv.append(v); pf.append(f); first.append(first[-1] + v.shape[0]); nfm.append(f.shape[0])
    s["packed_large"] = dict(vertices=np.concatenate(pv), first_idx=np.array(first, np.int64), faces=np.concatenate(pf),
                             num_faces=np.array(nfm, np.int64), N=250, key=0x0BAD_F00D, packed=True)
    return s


def _codes(rng, shape, dt):
    """Features and upstream gradients: multiples of 1/8 in [-2, 2], which compress well."""
    return (rng.integers(-16, 17, size=shape) / 8.0).astype(dt)


class _IeeeSqrt(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        out = torch.from_numpy(np.sqrt(x.detach().numpy()))
        ctx.save_for_backward(out)
        return out

    @staticmethod
    def backward(ctx, grad):
        out, = ctx.saved_tensors
        return grad / (2 * out)


class _Patched:
    """Categorical.sample -> the given choices (N, B); torch.rand -> u_raw, then v, as (B, N, 1)."""

    def __init__(self, choices, u, v):
        self.choices, self.rand = choices, [u, v]

    def __enter__(self):
        self._sample, self._rand = torch.distributions.Categorical.sample, torch.rand
        choices, queue = self.choices, self.rand

        def sample(dist, shape=torch.Size()):
            assert tuple(shape) == (choices.shape[1],)
            return torch.from_numpy(choices.T.copy())

        def rand(shape, device=None, dtype=None):
            x = queue.pop(0)
            assert tuple(shape) == x.shape + (1,) and x.dtype == np.dtype(str(dtype).replace("torch.", ""))
            return torch.from_numpy(x.copy())[..., None]

        torch.distributions.Categorical.sample = sample
        torch.rand = rand
        return self

    def __exit__(self, *exc):
        torch.distributions.Categorical.sample, torch.rand = self._sample, self._rand
        assert not self.rand or exc[0] is not None


def _check_margin(c, t):
    """No t within 4 F 2^-53 c_last of a CDF boundary (per view)."""
    F = c.shape[-1]
    tol = 4 * F * 2.0 ** -53 * c[-1]
    i = np.searchsorted(c, t)
    near = np.minimum(np.abs(c[np.clip(i, 0, F - 1)] - t), np.abs(c[np.clip(i - 1, 0, F - 1)] - t))
    assert (near > tol).all(), (near.min(), tol)


def _dense(tm, name, sc, dt, rng):
    v = sc["vertices"].astype(dt)
    faces = sc["faces"]
    B, N, D = v.shape[0], sc["N"], sc["D"]
    ff = _codes(rng, (B, faces.shape[0], 3, D), dt) if D else None
    given = sc.get("areas")
    given = None if given is None else given.astype(dt)
    pts, ch, feats, (r, u, v_), t = osp.sample_points(v, faces, N, sc["key"], areas=given, face_features=ff)
    areas_o = osp.face_areas(v, faces)
    c = osp.cdf(areas_o if given is None else given)
    for b in range(B):
        _check_margin(c[b], t[b])
    gp = _codes(rng, (B, N, 3), dt)
    gfeat = _codes(rng, (B, N, D), dt) if D else None
    ga = _codes(rng, (B, faces.shape[0]), dt)

    tv = torch.from_numpy(v).requires_grad_(True)
    tff = torch.from_numpy(ff).requires_grad_(True) if D else None
    tf = torch.from_numpy(faces)
    with _Patched(ch, u, v_):
        out = tm.sample_points(tv, tf, N, areas=None if given is None else torch.from_numpy(given), face_features=tff)
    rp, rch = out[0], out[1]
    loss = (rp * torch.from_numpy(gp)).sum()
    if D:
        loss = loss + (out[2] * torch.from_numpy(gfeat)).sum()
    loss.backward()
    assert np.array_equal(rch.numpy(), ch)
    assert np.array_equal(rp.detach().numpy(), pts), name
    if D:
        assert np.array_equal(out[2].detach().numpy(), feats), name
    ta = torch.from_numpy(v).requires_grad_(True)
    ra = tm.face_areas(ta, tf)
    ra.backward(torch.from_numpy(ga))
    assert np.array_equal(ra.detach().numpy(), areas_o), name
    rec = dict(vertices=v, faces=faces, key=np.int64(sc["key"]), N=np.int64(N), areas=ra.detach().numpy(),
               points=rp.detach().numpy(), choices=rch.numpy(), grad_points=gp, grad_areas=ga,
               ref_grad_vertices=tv.grad.numpy(), ref_grad_vertices_areas=ta.grad.numpy())
    if given is not None:
        rec["given_areas"] = given
    if D:
        rec.update(face_features=ff, features=out[2].detach().numpy(), grad_features=gfeat,
                   ref_grad_face_features=tff.grad.numpy())
    return rec


def _packed(tm, name, sc, dt, rng):
    v = sc["vertices"].astype(dt)
    faces, first, nfm, N = sc["faces"], sc["first_idx"], sc["num_faces"], sc["N"]
    B = nfm.shape[0]
    off = np.concatenate([[0], np.cumsum(nfm)])
    merged = faces + np.repeat(first[:-1], nfm)[:, None]
    areas_o = osp.face_areas(v[None], merged)[0]
    r, u, v_ = osp.uniforms(sc["key"], B, N, dt)
    ch = np.empty((B, N), np.int64)
    for b in range(B):
        c = osp.cdf(areas_o[off[b]:off[b + 1]])
        ch[b], t = osp.choose(c, r[b])
        _check_margin(c, t)
    w = osp.weights(u, v_)
    pts = osp.interpolate(w, *(v[merged[ch + off[:-1, None], k]] for k in range(3)))
    gp = _codes(rng, (B, N, 3), dt)
    ga = _codes(rng, (faces.shape[0],), dt)
    tv = torch.from_numpy(v).requires_grad_(True)
    args = (torch.from_numpy(first), torch.from_numpy(faces), torch.from_numpy(nfm))
    with _Patched(ch, u, v_):
        rp, rch = tm.packed_sample_points(tv, args[0], args[1], args[2], N)
    (rp * torch.from_numpy(gp)).sum().backward()
    assert np.array_equal(rch.numpy(), ch + off[:-1, None])
    assert np.array_equal(rp.detach().numpy(), pts), name
    ta = torch.from_numpy(v).requires_grad_(True)
    ra = tm.packed_face_areas(ta, *args)
    ra.backward(torch.from_numpy(ga))
    assert np.array_equal(ra.detach().numpy(), areas_o), name
    return dict(vertices=v, first_idx=first, faces=faces, num_faces=nfm, key=np.int64(sc["key"]), N=np.int64(N),
                areas=ra.detach().numpy(), points=rp.detach().numpy(), choices=rch.numpy(), grad_points=gp,
                grad_areas=ga, ref_grad_vertices=tv.grad.numpy(), ref_grad_vertices_areas=ta.grad.numpy())


def main():
    tm = ref_import.module("kaolin.ops.mesh.trianglemesh")
    torch.sqrt = _IeeeSqrt.apply
    rng = np.random.default_rng(2024)
    store = {}
    for name, sc in scenes().items():
        for tag, dt in DTYPES.items():
            rec = (_packed if sc.get("packed") else _dense)(tm, name, sc, dt, rng)
            for k, x in rec.items():
                x = np.asarray(x)
                if k in INDICES:
                    assert x.min() >= -2 ** 31 and x.max() < 2 ** 31
                    x = x.astype(np.int32)
                store[f"{name}/{tag}/{k}"] = x
            print(f"{name}/{tag}: ok")
    np.savez_compressed(OUT, **store)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
