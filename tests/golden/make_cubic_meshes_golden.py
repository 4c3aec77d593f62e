"""Regenerate tests/golden/cubic_meshes.npz from the reference's own
kaolin.ops.conversions.voxelgrids_to_cubic_meshes, run on the CPU through oracle/ref_import.py (needs
the reference sources).

Keys are ``<scene>__grid`` (the batch, in the dtype the function is called with) and
``<scene>__<tri|quad>__<v|f><view>``; faces are stored as int32 to keep the file small (the function
returns int64).  Every scene's voxel differences round to -1, 0 or 1, where the
library's contract and the reference agree bit for bit.  Grids stay at 24^3 or below: the reference is
slow on the CPU.

    python tests/golden/make_cubic_meshes_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

OUT = os.path.join(HERE, "cubic_meshes.npz")


def scenes():
    rng = np.random.default_rng(18)
    s = {}
    fixture = np.ones((4, 2, 2, 2), bool)            # the reference's TestVoxelgridsToCubicMeshes grids
    fixture[0] = False
    fixture[2, :, 0, 0] = False
    fixture[3, 0, 0, :] = False
    fixture[3, 0, 1, 0] = False
    fixture[3, 1, 1, 1] = False
    s["fixture"] = fixture
    s["single_voxel"] = np.ones((1, 1, 1, 1), np.float32)
    s["box_3x4x5"] = np.ones((1, 3, 4, 5), bool)
    s["checker_6"] = (np.indices((6, 6, 6)).sum(0) % 2 == 0)[None]
    for d in (0.1, 0.5, 0.9):
        tag = int(d * 100)
        s[f"random{tag}_1x1x7"] = rng.random((2, 1, 1, 7)) < d
        s[f"random{tag}_2x3x4"] = rng.random((2, 2, 3, 4)) < d
        s[f"random{tag}_9x5x7"] = rng.random((2, 9, 5, 7)) < d
    s["random50_24"] = rng.random((1, 24, 24, 24)) < 0.5
    s["quarters_f32"] = (rng.integers(0, 5, (2, 7, 6, 5)) / 4).astype(np.float32)
    binary = rng.random((2, 8, 9, 10)) < 0.5
    s["binary_bool"] = binary
    s["binary_u8"] = binary.astype(np.uint8)
    s["binary_f32"] = binary.astype(np.float32)
    batch = rng.random((4, 6, 7, 5)) < 0.4
    batch[1] = False
    s["batch4_empty_view1"] = batch
    return s


def main():
    from oracle import ref_import
    ref_import.setup()
    from kaolin.ops.conversions import voxelgrid as ref

    store = {}
    for name, grid in scenes().items():
        store[f"{name}__grid"] = grid
        for mode, tri in (("tri", True), ("quad", False)):
            verts, faces = ref.voxelgrids_to_cubic_meshes(torch.from_numpy(grid), is_trimesh=tri)
            for b, (v, f) in enumerate(zip(verts, faces)):
                assert v.dtype == torch.float32 and f.dtype == torch.int64
                store[f"{name}__{mode}__v{b}"] = v.numpy()
                store[f"{name}__{mode}__f{b}"] = f.numpy().astype(np.int32)
    np.savez_compressed(OUT, **store)
    print(f"wrote {OUT}: {len(store)} arrays")


if __name__ == "__main__":
    main()
