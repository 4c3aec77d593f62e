"""CPU-side checks of the boundary: the C-ABI library loads and exports every
symbol include/dibr_b200.h declares, argument errors are detected on the host
without a GPU, the Python layer mirrors the reference signatures, calls the
library through one helper and refuses to run without CUDA (no CPU fallback)."""
import ast
import ctypes
import inspect
import os
import re

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib, _C
from kaolin_b200.render.mesh import rasterize, dibr_soft_mask, dibr_rasterization

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "dibr_b200.h")).read()
    declared = set(re.findall(r"\b(dibr_b200_[a-z_0-9]+)\s*\(", hdr))
    assert {"dibr_b200_forward", "dibr_b200_backward", "dibr_b200_packed_rasterize_forward",
            "dibr_b200_rasterize_backward", "dibr_b200_soft_mask_forward",
            "dibr_b200_soft_mask_backward", "dibr_b200_workspace_bytes",
            "dibr_b200_version"} <= declared
    lib = _lib.lib()
    for name in declared:
        assert hasattr(lib, name), name
    assert set(_lib.SIGNATURES) == declared
    assert lib.dibr_b200_version() >= 200


def test_header_cites_reference_interfaces():
    hdr = open(os.path.join(ROOT, "include", "dibr_b200.h")).read()
    for cite in ("rasterization.h:23-32", "rasterization.h:34-41", "dibr_soft_mask.h:23-30",
                 "dibr_soft_mask.h:32-42", "bindings.cpp:111-115"):
        assert cite in hdr


def test_workspace_query_and_host_side_errors():
    lib = _lib.lib()
    n = lib.dibr_b200_workspace_bytes(32, 32 * 20480, 1024, 1024)
    assert 50e6 < n < 200e6
    assert lib.dibr_b200_workspace_bytes(0, 10, 64, 64) == 0          # bad batch
    assert lib.dibr_b200_workspace_bytes(1, 10, 20000, 64) == 0       # image too large
    # null pointers / bad sizes are rejected before any CUDA call (no GPU needed)
    st = lib.dibr_b200_forward(1, 4, 8, 8, 1, None, None, None, None, None, 1000.0, 1e-8, 3,
                               7000.0, 20.0, 30, None, None, None, None, None, 0, None)
    assert st == _lib.EINVAL
    st = lib.dibr_b200_forward(1, 4, 20000, 8, 1, None, None, None, None, None, 1000.0, 1e-8, 3,
                               7000.0, 20.0, 30, None, None, None, None, None, 0, None)
    assert st == _lib.ESIZE
    with pytest.raises(RuntimeError):
        _lib.check(st, "dibr_b200_forward")
    # float64 entry points: same host-side contract
    n64 = lib.dibr_b200_workspace_bytes_f64(4, 4 * 20480, 1024, 1024)
    assert 0 < n64 < 200e6
    assert lib.dibr_b200_workspace_bytes_f64(0, 10, 64, 64) == 0
    st = lib.dibr_b200_forward_f64(1, 4, 8, 8, 1, None, None, None, None, None, 1000.0, 1e-8, 3,
                                   7000.0, 20.0, 30, None, None, None, None, None, 0, None)
    assert st == _lib.EINVAL
    st = lib.dibr_b200_backward_f64(1, 4, 20000, 8, 1, None, None, None, None, None, None, None,
                                    1000.0, 1e-8, 7000.0, 20.0, 30, None, None, None, 0, 0, None)
    assert st == _lib.ESIZE
    # peer push: argument errors are host-side
    import ctypes
    arr = (ctypes.c_void_p * 1)(ctypes.c_void_p(4096))
    assert lib.dibr_b200_peer_push(None, 32, arr, 1, 0, 0, None) == _lib.EINVAL           # no source
    assert lib.dibr_b200_peer_push(ctypes.c_void_p(4096), 24, arr, 1, 0, 0, None) == _lib.EINVAL   # not 16-byte units
    assert lib.dibr_b200_peer_push(ctypes.c_void_p(4096), 32, arr, 17, 0, 0, None) == _lib.EINVAL  # > 16 destinations
    assert lib.dibr_b200_peer_push(ctypes.c_void_p(4096), 0, arr, 1, 0, 0, None) == 0              # nothing to do
    assert lib.dibr_b200_peer_push_multicast(ctypes.c_void_p(4096), 32, None, 0, 0, None) == _lib.EINVAL
    assert lib.dibr_b200_peer_push_multicast(ctypes.c_void_p(4096), 32, ctypes.c_void_p(4104), 0, 0, None) == _lib.EINVAL


def test_misaligned_pointers_are_rejected_on_the_host():
    """The fused entry points require 16-byte aligned tensor pointers and say so before any CUDA
    call: fake device addresses that are all aligned but one give EINVAL without a GPU."""
    lib = _lib.lib()
    B, F, H, W, D = 1, 4, 8, 8, 3
    ok, off = ctypes.c_void_p(1 << 20), ctypes.c_void_p((1 << 20) + 4)    # off: one fp32 element in

    def forward(entry, **bad):
        p = dict(fvz=ok, fvi=ok, ff=ok, fnz=ok, valid=None, feat=ok, idx=ok, w=None, soft=ok)
        p.update(bad)
        return getattr(lib, entry)(B, F, H, W, D, p["fvz"], p["fvi"], p["ff"], p["fnz"], p["valid"], 1000.0, 1e-8,
                                   3, 7000.0, 20.0, 30, p["feat"], p["idx"], p["w"], p["soft"], ok, 1 << 20, None)

    def backward(entry, **bad):
        p = dict(g=ok, gs=ok, idx=ok, w=ok, soft=ok, fvi=ok, ff=ok, gfvi=ok, gff=ok)
        p.update(bad)
        return getattr(lib, entry)(B, F, H, W, D, p["g"], p["gs"], p["idx"], p["w"], p["soft"], p["fvi"], p["ff"],
                                   1000.0, 1e-8, 7000.0, 20.0, 30, p["gfvi"], p["gff"], ok, 1 << 20, 0, None)

    for entry in ("dibr_b200_forward", "dibr_b200_forward_bf16"):
        for name in ("fvz", "fvi", "ff", "fnz", "valid", "feat", "idx", "w", "soft"):
            assert forward(entry, **{name: off}) == _lib.EINVAL, (entry, name)
    assert forward("dibr_b200_forward_f64", w=ok, fvi=off) == _lib.EINVAL
    for entry in ("dibr_b200_backward", "dibr_b200_backward_bf16", "dibr_b200_backward_f64"):
        for name in ("g", "gs", "idx", "w", "soft", "fvi", "ff", "gfvi", "gff"):
            assert backward(entry, **{name: off}) == _lib.EINVAL, (entry, name)
    st = lib.dibr_b200_backward_views(B, F, H, W, D, off, ok, ok, None, ok, ok, ok, 0, 1000.0, 1e-8, 7000.0, 20.0,
                                      30, ok, ok, ok, 1 << 20, 0, 0, 1, None)
    assert st == _lib.EINVAL
    st = lib.dibr_b200_rasterize_backward(B, F, H, W, D, off, ok, ok, ok, ok, 1e-8, ok, ok, None)
    assert st == _lib.EINVAL


def test_python_signatures_match_reference():
    """rasterization.py:373-381, dibr.py:75-76,119-122."""
    sig = inspect.signature(rasterize)
    assert list(sig.parameters) == ["height", "width", "face_vertices_z", "face_vertices_image",
                                    "face_features", "valid_faces", "multiplier", "eps", "backend"]
    assert sig.parameters["backend"].default == "cuda" and sig.parameters["eps"].default is None
    sig = inspect.signature(dibr_soft_mask)
    assert [(k, v.default) for k, v in sig.parameters.items()][2:] == [
        ("sigmainv", 7000), ("boxlen", 0.02), ("knum", 30), ("multiplier", 1000.)]
    sig = inspect.signature(dibr_rasterization)
    assert list(sig.parameters) == ["height", "width", "face_vertices_z", "face_vertices_image",
                                    "face_features", "face_normals_z", "sigmainv", "boxlen", "knum",
                                    "multiplier", "eps", "rast_backend"]
    for op in ("packed_rasterize_forward_cuda", "rasterize_backward_cuda",
               "dibr_soft_mask_forward_cuda", "dibr_soft_mask_backward_cuda"):
        assert callable(getattr(_C.render.mesh, op))          # bindings.cpp:111-115


def test_no_cpu_fallback():
    fvz = torch.zeros(1, 4, 3)
    fvi = torch.zeros(1, 4, 3, 2)
    ff = torch.zeros(1, 4, 3, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        rasterize(8, 8, fvz, fvi, ff)
    with pytest.raises(RuntimeError, match="CUDA"):
        dibr_rasterization(8, 8, fvz, fvi, ff, torch.zeros(1, 4))
    with pytest.raises(RuntimeError, match="CUDA"):
        dibr_soft_mask(fvi, torch.zeros(1, 8, 8, dtype=torch.long))
    with pytest.raises(RuntimeError):
        _C.render.mesh.rasterize_backward_cuda(torch.zeros(1, 8, 8, 2), torch.zeros(1, 8, 8, 2),
                                               torch.zeros(1, 8, 8, dtype=torch.long),
                                               torch.zeros(1, 8, 8, 3), fvi, ff, 1e-8)
    with pytest.raises(ValueError):
        rasterize(8, 8, fvz, fvi, ff, backend="nvdiffrast")


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "kaolin_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f
                assert "oracle/" not in src.replace("tests/", ""), f


def test_library_is_called_only_through_lib_call():
    """Work is enqueued only through ``_lib.call``, which makes the tensors' device current, passes
    its stream and checks the status.  Elsewhere in the package the library is asked only for sizes,
    its version and traces, and no stream or pointer is converted by hand."""
    pkg = os.path.join(ROOT, "kaolin_b200")
    query = re.compile(r"dibr_b200_(\w*workspace_bytes\w*|version|trace_begin|trace_end)$")
    found = []
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            path = os.path.join(dirpath, f)
            if not f.endswith(".py") or path == os.path.join(pkg, "_lib.py"):
                continue
            for node in ast.walk(ast.parse(open(path).read(), path)):
                where = f"{os.path.relpath(path, ROOT)}:{getattr(node, 'lineno', '?')}"
                if isinstance(node, ast.Attribute) and node.attr == "cuda_stream":
                    found.append(f"{where}: .cuda_stream")
                if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute):
                    name, owner = node.func.attr, node.func.value
                    if name.startswith("dibr_b200_") and not query.match(name):
                        found.append(f"{where}: {name}()")
                    if name == "c_void_p" and isinstance(owner, ast.Name) and owner.id == "ctypes":
                        found.append(f"{where}: ctypes.c_void_p()")
    assert not found, "\n".join(found)


def test_hit_cache_sizing_policy():
    """Every tile is cached when that fits in 4 GB (BASELINE configs[1]/[2]: a third of the tiles
    touch the silhouette at 256^2 - caching 1/8 of them halved the throughput), else as many as fit."""
    from kaolin_b200.render.mesh import _host
    lib = _lib.lib()
    assert _host.cache_tiles_for(8, 256, 256, 30) == 8 * 16 * 16                 # c2: all tiles
    c3 = _host.cache_tiles_for(64, 512, 512, 30)
    assert 0.5 * 64 * 1024 < c3 <= 64 * 1024                                      # c3: more than half
    c4 = _host.cache_tiles_for(32, 1024, 1024, 30)
    assert 0.25 * 32 * 4096 < c4 < 32 * 4096                                      # c4: the 4 GB cap
    base = lib.dibr_b200_workspace_bytes(32, 32 * 20480, 1024, 1024)
    full = lib.dibr_b200_workspace_bytes_cached(32, 32 * 20480, 1024, 1024, 30, c4)
    assert base < full <= base + _host.CACHE_MAX_BYTES + (1 << 20)
    assert _host.cache_tiles_for(1, 16, 16, 30) == 1
