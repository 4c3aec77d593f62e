"""CPU check that the weights the rasterize backward recomputes are the forward's bits.

The fused forward no longer stores the (B,H,W,3) barycentric weights; the backward
recomputes them for the face in face_idx with raster_weights_of (dibr_math.cuh).  For every
(pixel, face) pair that raster_weights reports inside, raster_weights_of must give the same
bits, and it must write all three weights for every other pair too.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from kaolin_b200 import synthetic

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_math", "known_face.cpp")
LIB = os.path.join(HERE, "host_math", "_build", "libknown_face.so")
_f = ctypes.POINTER(ctypes.c_float)
_b = ctypes.POINTER(ctypes.c_uint8)


@pytest.fixture(scope="module")
def kf():
    hdr = os.path.join(HERE, "..", "kaolin_b200", "csrc", "dibr_math.cuh")
    if (not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(SRC),
                                                               os.path.getmtime(hdr))):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC",
                               "-shared", "-o", LIB, SRC])
    return ctypes.CDLL(LIB)


def run(kf, H, W, fvi, multiplier, eps, fill=np.nan):
    xy = np.ascontiguousarray(fvi.reshape(-1, 3, 2) * np.float32(multiplier), dtype=np.float32)
    F = xy.shape[0]
    inside = np.empty((H, W, F), np.uint8)
    w_fwd = np.empty((H, W, F, 3), np.float32)
    w_of = np.full((H, W, F, 3), fill, np.float32)
    kf.hm_known_face_weights(H, W, F, xy.ctypes.data_as(_f), ctypes.c_float(multiplier), ctypes.c_float(eps),
                             inside.ctypes.data_as(_b), w_fwd.ctypes.data_as(_f), w_of.ctypes.data_as(_f))
    return inside.astype(bool), w_fwd, w_of


SCENES = [
    ("ico2", lambda: synthetic.icosphere_views(1, 2, seed=1)[1], 40, 36),
    ("soup", lambda: synthetic.triangle_soup(1, 120, seed=3, coverage=4.0)[1], 33, 29),
]


@pytest.mark.parametrize("multiplier", [1000.0, 100.0, 1.0, 3.7])
@pytest.mark.parametrize("name,gen,H,W", SCENES, ids=[s[0] for s in SCENES])
def test_recomputed_weights_are_the_forward_bits(kf, name, gen, H, W, multiplier):
    fvi = gen()[0]
    inside, w_fwd, w_of = run(kf, H, W, fvi, multiplier, 1e-8)
    assert inside.sum() > 100
    assert np.array_equal(w_fwd[inside].view(np.uint32), w_of[inside].view(np.uint32))


def test_degenerate_faces(kf):
    """Zero-area faces (the eps addition decides the sign), tiny and huge faces, and
    infinite or NaN coordinates: the recomputation still matches wherever the forward
    accepts the face, and writes every weight."""
    _, fvi, _ = synthetic.triangle_soup(1, 40, seed=9, coverage=6.0)
    fvi = fvi[0]
    extra = np.stack([
        np.full((3, 2), 0.3, np.float32),                                  # a point
        np.array([[0, 0], [0.5, 0.5], [1, 1]], np.float32),                # a segment
        np.array([[0, 0], [1e-7, 0], [0, 1e-7]], np.float32),              # below eps at multiplier 1
        np.array([[-1e30, -1e30], [1e30, -1e30], [0, 1e30]], np.float32),  # huge
        np.array([[np.inf, 0], [0, 1], [1, 0]], np.float32),
        np.array([[np.nan, 0], [0, 1], [1, 0]], np.float32),
    ])
    fvi = np.concatenate([fvi, extra, fvi[:5]], 0)
    for multiplier, eps in ((1000.0, 1e-8), (1.0, 1e-8), (1.0, 0.0), (1000.0, 1e-3)):
        for H, W in ((17, 23), (1, 1), (4, 64)):
            inside, w_fwd, w_of = run(kf, H, W, fvi, multiplier, eps)
            assert np.array_equal(w_fwd[inside].view(np.uint32), w_of[inside].view(np.uint32))
            _, _, w_of0 = run(kf, H, W, fvi, multiplier, eps, fill=0.0)
            assert np.array_equal(w_of.view(np.uint32), w_of0.view(np.uint32))   # nothing left unwritten
