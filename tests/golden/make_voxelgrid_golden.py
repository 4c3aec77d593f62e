"""Regenerate tests/golden/voxelgrid.npz from the reference's own kaolin.ops.voxelgrid functions, run on
the CPU through oracle/ref_import.py (needs the reference sources; its fill is scipy's
binary_fill_holes).

Keys are ``<function>__<scene>__<item>``: fill and odms scenes store ``grid`` and ``out``, surface
scenes ``grid``, ``wide`` and ``thin``, project scenes ``odms``, ``votes``, ``out`` and, unless the
grid is the default full one, ``grid``.  Non-binary float grids hold small dyadic values only, so
every window sum is exact in any order.

    python tests/golden/make_voxelgrid_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

OUT = os.path.join(HERE, "voxelgrid.npz")


def box(shape, lo, hi, grid=None, value=True):
    g = np.zeros(shape, bool) if grid is None else grid
    g[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = value
    return g


def shell(shape, lo, hi, grid=None):
    """A closed one-voxel shell between lo and hi (exclusive)."""
    g = box(shape, lo, hi, grid)
    return box(shape, [a + 1 for a in lo], [b - 1 for b in hi], g, False)


def serpentine(n):
    """A solid n^3 cube with a tunnel that winds back and forth through the x-y planes of z = n // 2 and
    leaves through the face x = 0."""
    g = np.ones((n, n, n), bool)
    z = n // 2
    g[0, 1, z] = False
    for x in range(1, n - 1, 2):
        g[x, 1:n - 1, z] = False
        if x + 1 < n - 1:
            y = n - 2 if (x // 2) % 2 == 0 else 1
            g[x + 1, y, z] = False
    return g


def spiral(n):
    """A solid n^3 cube with a tunnel that walks square rings of shrinking radius, one z level per ring,
    each ring joined to the next by a step up and a step inward; it reaches the face z = 0."""
    g = np.ones((n, n, n), bool)
    c = n // 2
    for k, r in enumerate(range(c - 1, 0, -1)):
        z = 1 + k
        g[c - r:c + r + 1, c - r, z] = g[c - r:c + r + 1, c + r, z] = False
        g[c - r, c - r:c + r + 1, z] = g[c + r, c - r:c + r + 1, z] = False
        if r > 1:
            g[c - r, c - r, z + 1] = g[c - r + 1, c - r, z + 1] = False
    g[c + c - 1, c, 0] = False
    return g


def fill_scenes(rng):
    s = {}
    s["doc"] = np.array([[[[0., 0., 0., 0., 0.], [0., 1., 1., 1., 1.], [0., 1., 1., 1., 1.], [0., 1., 1., 1., 1.]],
                          [[0., 0., 0., 0., 0.], [0., 1., 1., 1., 1.], [0., 1., 0., 0., 1.], [0., 1., 1., 1., 1.]],
                          [[0., 0., 0., 0., 0.], [0., 1., 1., 1., 1.], [0., 1., 1., 1., 1.], [0., 1., 1., 1., 1.]]]],
                        np.float32)
    s["cavity"] = shell((10, 10, 10), (2, 2, 2), (8, 8, 8))[None]
    n = shell((15, 15, 15), (1, 1, 1), (14, 14, 14))
    n = shell((15, 15, 15), (4, 4, 4), (11, 11, 11), n)
    s["nested"] = shell((15, 15, 15), (6, 6, 6), (9, 9, 9), n)[None]
    e = shell((9, 9, 9), (2, 2, 2), (7, 7, 7))
    e[2, 2, 4] = False              # an edge voxel of the shell: the cavity reaches it only diagonally
    s["leak_edge"] = e[None]
    c = shell((9, 9, 9), (2, 2, 2), (7, 7, 7))
    c[2, 2, 2] = False              # a corner voxel
    s["leak_corner"] = c[None]
    h = shell((9, 9, 9), (0, 0, 0), (9, 9, 9))
    h[0, 4, 4] = False              # a one-voxel hole in the border wall
    s["hole_to_border"] = h[None]
    w = np.zeros((11, 11, 11), bool)
    w[5] = True                     # a one-voxel wall across x, and a closed thin shell on each side
    w = shell((11, 11, 11), (1, 1, 1), (5, 5, 5), w)
    s["thin_walls"] = shell((11, 11, 11), (6, 6, 6), (11, 11, 11), w)[None]
    s["serpentine"] = serpentine(17)[None]
    s["spiral"] = spiral(15)[None]
    for side in (1, 2, 3):
        s[f"side{side}_random"] = rng.random((2, side, side, side)) < 0.5
        s[f"side{side}_full"] = np.ones((1, side, side, side), bool)
        s[f"side{side}_empty"] = np.zeros((1, side, side, side), bool)
    s["side3_ring"] = ~box((3, 3, 3), (1, 1, 1), (2, 2, 2))[None]
    s["noncubic_5x7x9"] = np.stack([rng.random((5, 7, 9)) < 0.6, shell((5, 7, 9), (0, 0, 0), (5, 7, 9))])
    big = shell((37, 64, 50), (3, 5, 7), (30, 60, 44))
    big = shell((37, 64, 50), (10, 20, 15), (20, 40, 30), big)
    big[3, 30, 20] = False
    s["noncubic_37x64x50"] = np.stack([big, rng.random((37, 64, 50)) < 0.69])
    for d in (0.3, 0.5, 0.69, 0.75, 0.85):
        s[f"random_{int(d * 100)}"] = rng.random((2, 24, 24, 24)) < d
    f = np.where(shell((8, 8, 8), (1, 1, 1), (7, 7, 7)), np.float32(1), np.float32(0))
    f[1, 3, 3], f[1, 4, 4], f[6, 3, 3], f[3, 1, 3] = np.nan, -2.5, np.float32(1e-45), -np.inf
    f[3, 3, 1] = -0.0               # a -0.0 in the wall opens the cavity
    g = f.copy()
    g[3, 3, 1] = np.float32(1.2e-38) / 4   # a subnormal keeps it closed
    s["float_special"] = np.stack([f, g])
    s["int64"] = (shell((8, 8, 8), (1, 1, 1), (7, 7, 7)).astype(np.int64) * -3)[None]
    s["float64"] = np.where(rng.random((2, 12, 12, 12)) < 0.69, rng.uniform(-2, 2, (2, 12, 12, 12)), 0.0)
    b3 = np.zeros((3, 10, 10, 10), bool)
    shell((10, 10, 10), (1, 1, 1), (9, 9, 9), b3[0])
    b3[1] = rng.random((10, 10, 10)) < 0.69
    shell((10, 10, 10), (0, 0, 0), (10, 10, 10), b3[2])
    b3[2, 0, 5, 5] = False
    s["batch3"] = b3
    return s


def surface_scenes(rng):
    s = {"doc": np.ones((1, 3, 3, 3), np.float32), "empty": np.zeros((1, 6, 6, 6), bool),
         "full": np.ones((2, 5, 6, 7), bool), "random_bool": rng.random((2, 9, 10, 11)) < 0.6,
         "random_f32": (rng.integers(0, 5, (2, 9, 10, 11)) / 4).astype(np.float32) * (rng.random((2, 9, 10, 11)) < 0.8),
         "random_f64": rng.integers(-4, 9, (2, 8, 8, 8)) / 8.0,
         "solid_f32": np.pad(np.ones((1, 6, 6, 6), np.float32), ((0, 0), (1, 1), (1, 1), (1, 1)))}
    return s


def odms_scenes(rng):
    doc = np.ones((2, 2, 2, 2), np.float32)
    doc[0, :, 0, :] = 0
    return {"doc": doc, "empty": np.zeros((1, 5, 5, 5), bool), "full": np.ones((1, 4, 4, 4), bool),
            "random": rng.random((2, 9, 9, 9)) < 0.1, "random_dense": rng.random((1, 33, 33, 33)) < 0.02,
            "side1": np.array([[[[1]]], [[[0]]]], np.uint8),
            "nan": np.where(rng.random((1, 6, 6, 6)) < 0.05, np.float32(np.nan), np.float32(0))}


def project_scenes(rng):
    s = {}
    doc = np.zeros((1, 6, 2, 2), np.float32)
    doc[0, 1, 1, 1] = 2
    s["doc_v1"] = dict(odms=doc, votes=1)
    s["doc_v2"] = dict(odms=doc, votes=2)
    D = 7
    base = rng.integers(0, D + 1, (2, 6, D, D))
    for votes in range(8):
        s[f"full_i64_v{votes}"] = dict(odms=base.astype(np.int64), votes=votes)
    occ = rng.random((2, D, D, D)) < 0.7
    s["bool_i32_v2"] = dict(odms=base.astype(np.int32), grid=occ, votes=2)
    s["bool_i64_v3"] = dict(odms=base.astype(np.int64), grid=occ, votes=3)
    s["f32_grid_f32_v1"] = dict(odms=base.astype(np.float32),
                                grid=(rng.integers(0, 9, (2, D, D, D)) / 4).astype(np.float32), votes=1)
    frac = (rng.integers(0, 4 * D + 4, (2, 6, D, D)) / 4 - 0.5)
    s["f64_grid_frac_f64_v2"] = dict(odms=frac, grid=rng.integers(-8, 9, (2, D, D, D)) / 8.0, votes=2)
    s["full_frac_f32_v1"] = dict(odms=frac.astype(np.float32), votes=1)
    s["full_frac_f64_v4"] = dict(odms=frac, votes=4)
    u8 = rng.integers(0, 4, (2, D, D, D)).astype(np.uint8)
    for votes in (1, 2, 7):
        s[f"u8_wrap_i64_v{votes}"] = dict(odms=base.astype(np.int64), grid=u8, votes=votes)
    s["u8_wrap_i32_v1"] = dict(odms=base.astype(np.int32), grid=np.ones((2, D, D, D), np.uint8), votes=1)
    s["empty_odms_full"] = dict(odms=np.zeros((1, 6, 4, 4), np.int64), votes=1)
    return s


def main():
    from oracle import ref_import
    ref_import.setup()
    from kaolin.ops import voxelgrid as ref

    rng = np.random.default_rng(16)
    store = {}
    for name, g in fill_scenes(rng).items():
        store[f"fill__{name}__grid"] = g
        store[f"fill__{name}__out"] = ref.fill(torch.from_numpy(g)).numpy()
    for name, g in surface_scenes(rng).items():
        store[f"surface__{name}__grid"] = g
        for mode in ("wide", "thin"):
            store[f"surface__{name}__{mode}"] = ref.extract_surface(torch.from_numpy(g), mode).numpy()
    for name, g in odms_scenes(rng).items():
        store[f"odms__{name}__grid"] = g
        store[f"odms__{name}__out"] = ref.extract_odms(torch.from_numpy(g)).numpy()
    for name, sc in project_scenes(rng).items():
        store[f"project__{name}__odms"] = sc["odms"]
        store[f"project__{name}__votes"] = np.int64(sc["votes"])
        grid = None
        if "grid" in sc:
            store[f"project__{name}__grid"] = sc["grid"]
            grid = torch.from_numpy(sc["grid"])
        store[f"project__{name}__out"] = ref.project_odms(torch.from_numpy(sc["odms"]), grid, sc["votes"]).numpy()
    np.savez_compressed(OUT, **store)
    print(f"wrote {OUT}: {len(store)} arrays")


if __name__ == "__main__":
    main()
