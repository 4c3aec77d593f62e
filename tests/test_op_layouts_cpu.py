"""The workspace layouts of every operator outside the rasterizer (kaolin_b200/csrc/op_layouts.h), checked
on a CPU.

The header is compiled as plain C++ (tests/host_math/op_layouts.cpp).  For every family, over shapes
that include zeros and the size limits of its entry points, and for a workspace pointer at every offset
from a 256-byte boundary: each piece starts on a 256-byte boundary, lies inside the workspace, overlaps
no other piece and holds what its kernels index; the workspace does not fit one byte short of the
total; and the library's size query returns the header's total.  Every entry point that carves a
workspace says EWORKSPACE one byte short of its size query, whatever the pointer's alignment.
"""
import ctypes
import json
import os
import subprocess
import sys

import pytest

from kaolin_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "host_math", "op_layouts.cpp")
HDR = os.path.join(ROOT, "kaolin_b200", "csrc", "op_layouts.h")
LIB = os.path.join(HERE, "host_math", "_build", "libop_layouts.so")
ALIGN = 256
BASE_PTR = 1 << 40          # a fake workspace address on a 256-byte boundary
INT32_MAX = (1 << 31) - 1
SCAN_TILE = 4096            # elements per tile sum of the exclusive scan
MAX_CELLS = 16              # grid cells a face is inserted in before it goes to the wide list
BWD_CTAS = 264              # the lighting backward's per-CTA partial slots

GRID = ["bounds", "counters", "cnt", "off", "entries", "wide"]
TOPO = ["count", "raw", "sums", "long_rows", "long_count"]
FAMILIES = {   # name: (id in ol_layout, pieces in its order)
    "deftet": (0, GRID),
    "check_sign_build": (1, ["maxlen"] + GRID + ["boxes", "records"]),
    "check_sign_query": (2, ["cnt", "off", "pcell", "order"]),
    "mesh_topology": (3, TOPO),
    "subdivision": (4, ["count", "sums"]),
    "tet_topology": (5, TOPO + ["corner_ptr", "corners", "degree", "weight", "status", "edge_ptr"]),
    "marching_tets": (6, ["flags", "sums"]),
    "marching_cubes": (7, ["counts", "sums"]),
    "lighting": (8, ["partial"]),
}


def grid_side(F):
    G = 8
    while G < 256 and G * G < F:
        G += 8
    return G


def scan_sums(n):
    """Bytes of tile sums the scan writes: one int per tile of SCAN_TILE elements."""
    return 4 * -(-n // SCAN_TILE)


def grid_needs(B, F):
    cells = 4 * B * (grid_side(F) ** 2 + 1)
    return {"bounds": 16 * B, "counters": 2 * cells, "cnt": cells, "off": cells,
            "entries": 4 * B * F * MAX_CELLS, "wide": 4 * B * F}


def topo_needs(V, corners, R):
    return {"count": 4 * V, "raw": 4 * R * corners, "sums": scan_sums(V), "long_rows": 4 * V, "long_count": 4}


# The bytes each piece's kernels index, from the family's arguments.
NEEDS = {
    "deftet": grid_needs,
    "check_sign_build": lambda B, F, ts: dict(grid_needs(B, F), maxlen=B * ts, boxes=16 * B * F, records=9 * ts * B * F),
    "check_sign_query": lambda B, F, N: {"cnt": 4 * B * (grid_side(F) ** 2 + 1), "off": 4 * B * (grid_side(F) ** 2 + 1),
                                         "pcell": 4 * B * N, "order": 4 * B * N},
    "mesh_topology": lambda V, F, S: topo_needs(V, F * S, 2),
    "subdivision": lambda V: {"count": 4 * V, "sums": scan_sums(V)},
    "tet_topology": lambda V, T: dict(topo_needs(V, 4 * T, 3), corner_ptr=4 * (V + 1), corners=16 * T, degree=4 * V,
                                      weight=4 * V, status=8, edge_ptr=4 * (V + 1)),
    "marching_tets": lambda B, E, T: {"flags": 4 * B * (E + 2 * T), "sums": scan_sums(B * (E + 2 * T))},
    "marching_cubes": lambda cubes: {"counts": 8 * cubes, "sums": scan_sums(cubes)},
    "lighting": lambda slots, floats, L: {"partial": 4 * slots * floats * L},
}

# (B, F, N) of check_sign: B F kMaxCells and B N stay below 2^31 - 1
CHECK_SIGN = [(1, 0, 0), (1, 0, 1), (1, 1, 1), (3, 1000, 5000), (7, 4097, 1), (1, 134217727, 2147483646),
              (16, 8388607, 10), (2, 10, 1073741823)]
V_EDGES = [0, 1, 4095, 4096, 4097, INT32_MAX - 1]
SHAPES = {
    "deftet": [(B, F) for B in (1, 3, 1000) for F in (0, 1, 64, 65, 5000, 65536, 65537, 134217727)],
    "check_sign_build": [(B, F, ts) for B, F, _ in CHECK_SIGN for ts in (4, 8)],
    "check_sign_query": CHECK_SIGN,
    # 2 F S < 2^31
    "mesh_topology": [(V, F, S) for V in V_EDGES
                      for F, S in ((0, 3), (1, 3), (5, 4), (INT32_MAX // 6, 3), (INT32_MAX // 14, 7))],
    "subdivision": [(V,) for V in V_EDGES],
    # 12 T < 2^31
    "tet_topology": [(V, T) for V in V_EDGES for T in (0, 1, 7, INT32_MAX // 12)],
    # B (E + 2 T) < 2^31 - 1
    "marching_tets": [(0, 0, 0), (1, 0, 0), (1, 6, 1), (3, 1000, 400), (1, 0, INT32_MAX // 12), (1, INT32_MAX - 1, 0),
                      (7, 1000, 4000)],
    # B N <= (2^31 - 1) / 5
    "marching_cubes": [(n,) for n in (0, 1, 4095, 4096, 4097, 2 * 258 ** 3, INT32_MAX // 5)],
    "lighting": [(BWD_CTAS, f, L) for f in (7, 9) for L in (0, 1, 64, 65, 1000, 1 << 20)],
}


@pytest.fixture(scope="module")
def ol():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(SRC), os.path.getmtime(HDR)):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", LIB, SRC])
    lib = ctypes.CDLL(LIB)
    lib.ol_layout.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int64)]
    lib.ol_carve.argtypes = [ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint64]
    lib.ol_carve.restype = ctypes.c_int64
    return lib


def layout(ol, family, *args):
    """(total bytes, {piece: (offset from the origin, bytes)}) of the header's layout."""
    fid, names = FAMILIES[family]
    out = (ctypes.c_int64 * 64)()
    assert ol.ol_layout(fid, (ctypes.c_int64 * 4)(*args), out) == 1 + 2 * len(names)
    return out[0], {name: (out[1 + 2 * i], out[2 + 2 * i]) for i, name in enumerate(names)}


@pytest.mark.parametrize("family", list(FAMILIES))
def test_every_piece_is_aligned_apart_and_inside(ol, family):
    for args in SHAPES[family]:
        total, pieces = layout(ol, family, *args)
        for name, need in NEEDS[family](*args).items():
            assert pieces[name][1] >= need, (family, args, name)
        top = dict(pieces)
        if "counters" in pieces:
            # one memset clears the grid's cnt and off: both lie in the counters piece, apart
            at, n = pieces["counters"]
            cnt, off = top.pop("cnt"), top.pop("off")
            assert at == cnt[0] and cnt[0] + cnt[1] <= off[0] and off[0] + off[1] <= at + n, (family, args)
            assert off[0] % ALIGN == 0, (family, args)
        spans = sorted((at, at + n, name) for name, (at, n) in top.items() if n > 0)
        for (_, e0, a), (s1, _, b) in zip(spans, spans[1:]):
            assert e0 <= s1, (family, args, a, b)
        for offset in range(ALIGN):
            ws = BASE_PTR + offset
            origin = ol.ol_carve(ws, total, total)
            assert 0 <= origin < ALIGN and (ws + origin) % ALIGN == 0, (family, args, offset)
            for name, (at, n) in top.items():
                assert (ws + origin + at) % ALIGN == 0, (family, args, offset, name)
                assert origin + at + n <= total, (family, args, offset, name)
            assert ol.ol_carve(ws, total - 1, total) == -1, (family, args, offset)
        assert ol.ol_carve(0, 1 << 62, total) == -1             # no workspace


def total(ol, family, *args):
    return layout(ol, family, *args)[0]


def test_size_queries_return_the_header_totals(ol):
    lib = _lib.lib()
    for B, F in SHAPES["deftet"]:
        assert lib.dibr_b200_deftet_workspace_bytes(B, F) == total(ol, "deftet", B, F), (B, F)
    for B, F, N in CHECK_SIGN:
        for dtype, ts in ((_lib.DTYPE_F32, 4), (_lib.DTYPE_F64, 8)):
            build, query = _lib.check_sign_workspace_bytes(B, F, N, dtype, "check_sign")
            assert build == total(ol, "check_sign_build", B, F, ts), (B, F, ts)
            assert query == total(ol, "check_sign_query", B, F, N), (B, F, N)
    for V, F, S in SHAPES["mesh_topology"]:
        assert lib.dibr_b200_mesh_topology_workspace_bytes(V, F, S) == total(ol, "mesh_topology", V, F, S), (V, F, S)
    for (V,) in SHAPES["subdivision"]:
        for F in (0, 1, 5, INT32_MAX // 6):
            assert lib.dibr_b200_loop_subdivision_workspace_bytes(V, F) == total(ol, "subdivision", V), (V, F)
    for V, T in SHAPES["tet_topology"]:
        assert lib.dibr_b200_tet_topology_workspace_bytes(V, T) == total(ol, "tet_topology", V, T), (V, T)
    for B, E, T in SHAPES["marching_tets"]:
        assert lib.dibr_b200_marching_tets_workspace_bytes(B, E, T) == total(ol, "marching_tets", B, E, T), (B, E, T)
    for B, X, Y, Z, pad in ((0, 3, 3, 3, 1), (1, 1, 1, 1, 0), (2, 256, 256, 256, 1), (1, 754, 754, 754, 0),
                            (3, 5, 7, 9, 0), (25, 256, 256, 256, 1)):
        out = ctypes.c_size_t(0)
        assert lib.dibr_b200_marching_cubes_workspace_bytes(B, X, Y, Z, pad, ctypes.byref(out)) == 0
        cubes = B * (X + 2 * pad) * (Y + 2 * pad) * (Z + 2 * pad)
        assert out.value == total(ol, "marching_cubes", cubes), (B, X, Y, Z, pad)
    for L in (0, 1, 64, 65, 1000, 1 << 20):
        sg = total(ol, "lighting", BWD_CTAS, 7, L)
        assert lib.dibr_b200_sg_inner_product_workspace_bytes(L) == sg, L
        assert lib.dibr_b200_diffuse_workspace_bytes(_lib.LIGHT_SG_INNER_PRODUCT, L) == sg, L
        assert lib.dibr_b200_diffuse_workspace_bytes(_lib.LIGHT_SG_FITTED, L) == sg, L
        assert lib.dibr_b200_specular_workspace_bytes(L) == sg, L
        assert lib.dibr_b200_sg_shade_workspace_bytes(L) == sg, L
    assert lib.dibr_b200_diffuse_workspace_bytes(_lib.LIGHT_SH9, 1) == total(ol, "lighting", BWD_CTAS, 9, 1)


# Runs in a process that sees no CUDA device: fake pointers reach only the host-side checks, and a call
# that passes them fails at its first CUDA call.
ENTRY_POINTS = r"""
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
import torch
from kaolin_b200 import _lib
assert torch.cuda.device_count() == 0, "the fake pointers below must not reach a device"
lib = _lib.lib()
p = 1 << 32                     # a fake device pointer, 256-byte aligned
q = p + (1 << 24)               # another, for a second workspace
B, F, N, V, E, L = 2, 100, 50, 40, 120, 3
build, query = _lib.check_sign_workspace_bytes(B, F, N, _lib.DTYPE_F32, "check_sign")
build1, query1 = _lib.check_sign_workspace_bytes(1, F, N, _lib.DTYPE_F64, "check_sign")
calls = {   # name: (workspace bytes, call(workspace, workspace_bytes))
    "deftet_sparse_render_forward": (lib.dibr_b200_deftet_workspace_bytes(B, F), lambda ws, n:
        lib.dibr_b200_deftet_sparse_render_forward(B, F, 64, 4, p, p, p, p, p, 1e-8, p, p, p, p, ws, n, None)),
    "check_sign_build": (build, lambda ws, n: lib.dibr_b200_check_sign_build(B, V, F, 0, p, p, p, ws, n, None)),
    "check_sign_query(mesh)": (build, lambda ws, n:
        lib.dibr_b200_check_sign_query(B, F, N, 0, p, ws, n, p, q, query, None)),
    "check_sign_query": (query, lambda ws, n: lib.dibr_b200_check_sign_query(B, F, N, 0, p, q, build, p, ws, n, None)),
    "mesh_intersection_count": (build1 + query1, lambda ws, n:
        lib.dibr_b200_mesh_intersection_count(F, N, 1, p, p, p, p, p, ws, n, None)),
    "mesh_topology_build": (lib.dibr_b200_mesh_topology_workspace_bytes(V, F, 3), lambda ws, n:
        lib.dibr_b200_mesh_topology_build(V, F, 3, *[p] * 8, ws, n, None)),
    "loop_subdivision_build": (lib.dibr_b200_loop_subdivision_workspace_bytes(V, F), lambda ws, n:
        lib.dibr_b200_loop_subdivision_build(V, F, *[p] * 11, ws, n, None)),
    "tet_topology_build": (lib.dibr_b200_tet_topology_workspace_bytes(V, F), lambda ws, n:
        lib.dibr_b200_tet_topology_build(V, F, *[p] * 7, ws, n, None)),
    "marching_tets_count": (lib.dibr_b200_marching_tets_workspace_bytes(B, E, F), lambda ws, n:
        lib.dibr_b200_marching_tets_count(B, V, E, F, *[p] * 5, ws, n, None)),
    "marching_cubes_count": (_lib.marching_cubes_workspace_bytes(B, 5, 6, 7, 1, "marching_cubes"), lambda ws, n:
        lib.dibr_b200_marching_cubes_count(B, 5, 6, 7, 1, _lib.DTYPE_F32, p, 210, 42, 7, 1, 0.5, p, p, p, ws, n, None)),
    "sg_inner_product_backward": (lib.dibr_b200_sg_inner_product_workspace_bytes(L), lambda ws, n:
        lib.dibr_b200_sg_inner_product_backward(1000, L, *[p] * 13, ws, n, None)),
    "specular_backward": (lib.dibr_b200_specular_workspace_bytes(L), lambda ws, n:
        lib.dibr_b200_specular_backward(1000, L, *[p] * 15, ws, n, None)),
    "sg_shade_backward": (lib.dibr_b200_sg_shade_workspace_bytes(L), lambda ws, n:
        lib.dibr_b200_sg_shade_backward(B, 16, 24, L, *[p] * 19, ws, n, None)),
}
for model in (_lib.LIGHT_SG_INNER_PRODUCT, _lib.LIGHT_SG_FITTED, _lib.LIGHT_SH9):
    lights = 1 if model == _lib.LIGHT_SH9 else L
    calls[f"diffuse_backward({model})"] = (lib.dibr_b200_diffuse_workspace_bytes(model, lights), lambda ws, n, m=model,
        l=lights: lib.dibr_b200_diffuse_backward(m, 1000, l, *[p] * 11, ws, n, None))
ws = p + (1 << 28)
out = {name: [[call(ws + off, need - 1), call(ws + off, need)] for off in (0, 1, 3, 128, 255)]
       for name, (need, call) in calls.items()}
print(json.dumps(out))
"""


def test_entry_points_need_their_size_query():
    """Each entry point that carves a workspace says EWORKSPACE one byte short of its size query, from any
    pointer alignment, and passes the workspace check (and every other) at the size query."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    run = subprocess.run([sys.executable, "-c", ENTRY_POINTS, ROOT], env=env, capture_output=True, text=True,
                         timeout=300)
    assert run.returncode == 0, run.stderr
    got = json.loads(run.stdout.strip().splitlines()[-1])
    assert len(got) == 16
    for name, per_offset in got.items():
        for short, enough in per_offset:
            assert short == _lib.EWORKSPACE, (name, short)
            assert enough not in (_lib.EWORKSPACE, _lib.EINVAL, _lib.ESIZE), (name, enough)
