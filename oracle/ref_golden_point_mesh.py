"""TEST INFRASTRUCTURE — the scenes of the point-to-mesh distance tests and the stored outputs of the
reference's CUDA operators on them (``unbatched_triangle_distance_{forward,backward}_cuda``,
oracle/build_ref_point_mesh.py), kept whole in ``tests/golden/ref_cuda_point_mesh.npz`` so that the tests
need neither the reference's sources nor a build of them.

Each scene runs through the reference wrapper's steps (trianglemesh.py:87-99, 125-149), view by view:
zero-filled outputs, the forward, then zero-filled gradients and the backward with the scene's
``grad_dist``; in float32 and in float64.

Record on a GPU with oracle/_ref built:  KAOLIN_REF_CUDA_RECORD=1 python -m oracle.ref_golden_point_mesh
"""
import os
import sys

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                    "ref_cuda_point_mesh.npz")
OUTPUTS = ("dist", "face_idx", "dist_type", "grad_points", "grad_face_vertices")
DTYPES = {"f32": np.float32, "f64": np.float64}
# Scenes with a NaN face at an index that is a multiple of 512 (0 included): the documented deviation.
DEVIATION = ("degenerate_at_0", "degenerate_at_512")

_TRI = np.array([[0., 0., 0.], [1., 0., 0.], [0., 1., 0.]])


def _far_faces(rng, n, offset=50.0):
    """n random small faces far away from the origin (they never win)."""
    c = rng.normal(size=(n, 1, 3)) + offset
    return c + 0.3 * rng.normal(size=(n, 3, 3))


def _scene(points, faces, rng):
    points = np.asarray(points, np.float64)
    faces = np.asarray(faces, np.float64)
    if points.ndim == 2:
        points, faces = points[None], faces[None]
    grad = rng.normal(size=points.shape[:2])
    return points, faces, grad


def scenes():
    """name -> (points (B, N, 3), face_vertices (B, F, 3, 3), grad_dist (B, N)), float64 numpy."""
    rng = np.random.default_rng(1234)
    out = {}
    out["docstring"] = _scene([[0.5, 0.5, 0.5], [3., 4., 5.]], [[[0., 0., 0.], [0., 1., 0.], [0., 0., 1.]]], rng)
    # one point of each type against the triangle (0,0,0) (1,0,0) (0,1,0)
    out["types"] = _scene([[0.2, 0.2, 1.0], [-1., -1., 0.5], [2., -0.5, 0.3], [-0.5, 2., 0.3], [0.5, -1., 0.2],
                           [1., 1., 0.1], [-1., 0.5, 0.2]], _TRI[None], rng)
    # points exactly on vertices, on edges, in the plane, at u = 0 and u = 1
    exact = [[0, 0, 0], [1, 0, 0], [0, 1, 0], [0.5, 0, 0], [0.5, 0.5, 0], [0, 0.5, 0], [0.25, 0.25, 0],
             [0.25, 0.25, 0.5], [2, 0, 0], [-1, 0, 0], [0, 2, 0], [0, -1, 0], [0, 0, 1], [1, 0, 1], [0, 1, -1],
             [0.5, -0.5, 0], [0.75, 0.25, 0], [1, 1, 0], [-0.5, -0.5, 0]]
    out["exact"] = _scene(exact, _TRI[None], rng)
    # duplicate faces, and a fan around (0, 0, 0) whose faces are all equidistant from points on the axis
    dup = np.repeat(_TRI[None], 16, 0)
    out["duplicates"] = _scene(rng.normal(size=(64, 3)), dup, rng)
    ang = np.linspace(0, 2 * np.pi, 13)[:-1]
    fan = np.stack([np.zeros((12, 3)), np.stack([np.cos(ang), np.sin(ang), 0 * ang], 1),
                    np.stack([np.cos(np.roll(ang, -1)), np.sin(np.roll(ang, -1)), 0 * ang], 1)], 1)
    axis = np.stack([0 * ang[:8], 0 * ang[:8], np.linspace(-2, 2, 8)], 1)
    out["fan"] = _scene(np.concatenate([axis, rng.normal(size=(56, 3))]), fan, rng)
    # F around the reference's 512-face tile: ties that straddle index 511/512
    for F in (511, 512, 513, 1025):
        faces = _far_faces(rng, F)
        for k in (0, 255, 510, 511, 512, 1024):
            if k < F:
                faces[k] = _TRI + np.array([0., 0., 0.])
        pts = np.concatenate([rng.uniform(-0.5, 1.5, size=(48, 3)), [[0.2, 0.2, 0.7], [-1, -1, 0]]])
        out[f"tiles_{F}"] = _scene(pts, faces, rng)
    # degenerate faces (coincident, collinear, two coincident vertices) at index 3, 512 and 0
    degen = [np.zeros((3, 3)) + 0.5, np.array([[0., 0., 0.], [1., 1., 1.], [2., 2., 2.]]),
             np.array([[0., 0., 0.], [0., 0., 0.], [1., 0.5, 0.]])]
    for at, F in ((3, 16), (512, 600), (0, 16)):
        faces = _far_faces(rng, F, offset=3.0)
        for j, d in enumerate(degen):
            faces[at + 5 * j] = d
        pts = np.concatenate([rng.normal(size=(40, 3)), [[-1., -1., -1.], [3., 3., 3.], [-0.5, 0., 0.]]])
        out[f"degenerate_at_{at}"] = _scene(pts, faces, rng)
    # NaN, +-inf, +-3e38 and subnormal coordinates, in points and in vertices
    specials = [np.nan, np.inf, -np.inf, 3e38, -3e38, 1e-40, -1e-40, 1e-310]
    pts = rng.normal(size=(24, 3))
    for j, s in enumerate(specials):
        pts[j, j % 3] = s
    faces = rng.normal(size=(12, 3, 3))
    out["special_points"] = _scene(pts, faces, rng)
    faces = rng.normal(size=(24, 3, 3))
    for j, s in enumerate(specials):
        faces[2 * j + 1, j % 3, (j + 1) % 3] = s
    out["special_vertices"] = _scene(rng.normal(size=(32, 3)), faces, rng)
    # randn scenes at the sizes of the reference's test
    for B in (1, 3):
        for N in (11, 1025):
            for F in (11, 1025):
                out[f"randn_b{B}_n{N}_f{F}"] = _scene(rng.normal(size=(B, N, 3)), rng.normal(size=(B, F, 3, 3)), rng)
    # a noisy icosphere with points near its surface
    from kaolin_b200 import synthetic
    v, f = synthetic.icosphere(3)
    v = v + 0.01 * rng.normal(size=v.shape)
    d = rng.normal(size=(2000, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    out["icosphere"] = _scene(d * (1 + 0.05 * rng.normal(size=(2000, 1))), v[f], rng)
    return out


def run_reference(ext, points, faces, grad, dtype):
    """The reference wrapper's steps, view by view, on the GPU -> dict of numpy outputs (B, ...)."""
    import torch
    dev = torch.device("cuda")
    res = {k: [] for k in OUTPUTS}
    for b in range(points.shape[0]):
        p = torch.from_numpy(points[b].astype(dtype)).to(dev)
        fv = torch.from_numpy(faces[b].astype(dtype)).to(dev)
        g = torch.from_numpy(grad[b].astype(dtype)).to(dev)
        n = p.shape[0]
        dist = torch.zeros((n,), device=dev, dtype=p.dtype)
        idx = torch.zeros((n,), device=dev, dtype=torch.long)
        typ = torch.zeros((n,), device=dev, dtype=torch.int32)
        ext.unbatched_triangle_distance_forward_cuda(p, fv, dist, idx, typ)
        gp, gf = torch.zeros_like(p), torch.zeros_like(fv)
        ext.unbatched_triangle_distance_backward_cuda(g, p, fv, idx, typ, gp, gf)
        for k, t in zip(OUTPUTS, (dist, idx, typ, gp, gf)):
            res[k].append(t.cpu().numpy())
    return {k: np.stack(v) for k, v in res.items()}


def load():
    """{(scene, dtype name): {output: array}} from the store."""
    out = {}
    with np.load(PATH) as z:
        for k in z.files:
            scene, dt, name = k.rsplit(".", 2)
            out.setdefault((scene, dt), {})[name] = z[k]
    return out


def record():
    from . import build_ref_point_mesh
    ext = build_ref_point_mesh.load()
    assert ext is not None, "oracle/_ref/kaolin_ref_point_mesh_C.so is not built"
    flat = {}
    for name, (points, faces, grad) in scenes().items():
        for dt, dtype in DTYPES.items():
            for k, v in run_reference(ext, points, faces, grad, dtype).items():
                flat[f"{name}.{dt}.{k}"] = v
    np.savez_compressed(PATH, **flat)
    print(f"[ref_golden_point_mesh] {len(flat)} arrays -> {PATH}")


if __name__ == "__main__":
    if os.environ.get("KAOLIN_REF_CUDA_RECORD") != "1":
        sys.exit("set KAOLIN_REF_CUDA_RECORD=1 to record")
    record()
