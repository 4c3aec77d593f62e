"""Regenerate tests/golden/pointcloud.npz from the reference's own kaolin.ops.pointcloud.center_points, run
on the CPU through oracle/ref_import.py (needs the reference sources; its module imports warp, which
the import shim stubs).  The reference's farthest_point_sampling needs Warp and is not recorded.

Keys are ``center__<scene>__<item>``: ``points``, ``eps`` and the outputs ``plain`` (normalize=False)
and ``normalized`` (normalize=True).

    python tests/golden/make_pointcloud_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

OUT = os.path.join(HERE, "pointcloud.npz")


def scenes():
    g = torch.Generator().manual_seed(17)
    out = {}
    base = torch.rand((3, 200, 3), generator=g, dtype=torch.float64)
    out["scaled_translated"] = (base * torch.tensor([3.0, 0.25, 40.0], dtype=torch.float64)
                                + torch.tensor([-7.5, 1e3, 0.125], dtype=torch.float64), 1e-6)
    flat = torch.randn((2, 97, 3), generator=g, dtype=torch.float64)
    flat[..., 1] = 2.5                                           # a zero-range axis
    out["zero_range_axis"] = (flat, 1e-6)
    degenerate = torch.randn((2, 33, 3), generator=g, dtype=torch.float64)
    degenerate[1] = torch.tensor([0.5, -1.25, 3.0], dtype=torch.float64)   # every point the same
    out["degenerate_view"] = (degenerate, 1e-6)
    nan = torch.randn((2, 64, 3), generator=g, dtype=torch.float64)
    nan[0, 5, 2] = float("nan")
    nan[1, 0] = float("nan")
    out["nan_points"] = (nan, 1e-6)
    out["tiny_extent_eps"] = (1e-4 * torch.randn((2, 50, 3), generator=g, dtype=torch.float64), 1e-2)
    out["large_eps"] = (torch.randn((1, 40, 3), generator=g, dtype=torch.float64), 10.0)
    out["wide_channels"] = (torch.randn((2, 30, 6), generator=g, dtype=torch.float64) * 5, 1e-6)
    out["single_point"] = (torch.randn((4, 1, 3), generator=g, dtype=torch.float64), 1e-6)
    return out


def main():
    from oracle import ref_import
    ref = ref_import.module("kaolin.ops.pointcloud")
    store = {}
    for name, (pts64, eps) in scenes().items():
        for dt in (torch.float16, torch.float32, torch.float64):
            pts = pts64.to(dt)
            key = f"center__{name}_{str(dt).split('.')[-1]}"
            store[f"{key}__points"] = pts.numpy()
            store[f"{key}__eps"] = np.float64(eps)
            store[f"{key}__plain"] = ref.center_points(pts.clone()).numpy()
            store[f"{key}__normalized"] = ref.center_points(pts.clone(), normalize=True, eps=eps).numpy()
    np.savez_compressed(OUT, **store)
    print(f"wrote {OUT}: {len(store)} arrays")


if __name__ == "__main__":
    main()
