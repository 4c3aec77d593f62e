"""Writes tests/golden/check_sign.npz from the reference's own check_sign test
(tests/python/kaolin/ops/mesh/test_check_sign.py, read in place): its fixtures as data.

    verts (2, 8, 3) float64     the fixture's mesh and its negation (cat([verts, -verts]))
    faces (12, 3) int64
    zero_area_faces (4, 3)      the degenerate faces test_faces_with_zero_area appends
    points (2, 33, 3) float64   the 33 points and cat([points, flip(-points, dims=(1,))])
    expected (2, 33) bool       the expected output and its flip

float32 cases round these float64 values, as torch.tensor(..., dtype=torch.float) rounds the literals.

    python tests/golden/make_check_sign_golden.py
"""
import ast
import os
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402

REF_TEST = os.path.join(ref_import.REF, "tests", "python", "kaolin", "ops", "mesh", "test_check_sign.py")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "check_sign.npz")


def literals():
    """Every torch.tensor(<list literal>, ...) of TestCheckSign, by the function that holds it."""
    tree = ast.parse(open(REF_TEST).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "TestCheckSign")
    out = {}
    for fn in cls.body:
        if not isinstance(fn, ast.FunctionDef):
            continue
        for node in ast.walk(fn):
            if (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "tensor"
                    and node.args and isinstance(node.args[0], ast.List)):
                out.setdefault(fn.name, []).append(ast.literal_eval(node.args[0]))
    return out


def main():
    lit = literals()
    verts = np.array(lit["verts"][0], dtype=np.float64)
    points = np.array(lit["points"][0], dtype=np.float64)
    expected = np.array(lit["expected"][0], dtype=bool)
    np.savez_compressed(
        OUT,
        verts=np.concatenate([verts, -verts], axis=0),
        faces=np.array(lit["faces"][0], dtype=np.int64),
        zero_area_faces=np.array(lit["test_faces_with_zero_area"][0], dtype=np.int64),
        points=np.concatenate([points, np.flip(-points, axis=1)], axis=0),
        expected=np.concatenate([expected, np.flip(expected, axis=1)], axis=0))
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
