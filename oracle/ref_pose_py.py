"""ctypes wrapper over oracle/_ref/libref_pose_<variant>.so — the REFERENCE'S OWN grad_cost_p, compiled where it lies
(oracle/ref_pose_shim.cpp, oracle/ref_extract_pose.py).  TEST INFRASTRUCTURE ONLY.

The libraries exist only where the reference tree does; the tests that compare against them read the recorded outputs in
tests/golden/ref_pin_pose.npz elsewhere (tests/golden/make_pose_golden.py writes it).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import native

dp = C.POINTER(C.c_double)


def available(variant: str = "portable") -> bool:
    return native.available(f"_ref/libref_pose_{variant}.so")


def lib(variant: str = "portable"):
    return native.load(f"_ref/libref_pose_{variant}.so", _declare)


def _declare(L):
    L.rp_variant.restype = C.c_char_p
    L.rp_grad_cost_p.argtypes = [C.c_char_p, dp, dp, C.c_int, C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, dp, C.c_double, dp,
                                 C.c_double, C.c_int64, dp, dp]


def grad_cost_p(shape, poly_params, occ, lo, res, half, safety_hor, poses, polygon=None, variant="portable"):
    """The reference's grad_cost_p at poses [n, 3] against the map occ [X, Y, Z] (bool) at lo, voxel edge res: [n, 4] records
    (costp, gradp_x, gradp_y, grad_yaw)."""
    occ = np.ascontiguousarray(occ, dtype=np.uint8)
    X, Y, Z = occ.shape
    poses = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 3)
    pp = np.ascontiguousarray(poly_params, dtype=np.float64)
    lo = np.ascontiguousarray(lo, dtype=np.float64)
    half = np.ascontiguousarray(half, dtype=np.float64) * np.ones(3)
    poly = np.ascontiguousarray(polygon, dtype=np.float64).reshape(-1) if polygon is not None else None
    out = np.zeros((poses.shape[0], 4))
    p = lambda a: a.ctypes.data_as(dp) if a is not None else None  # noqa: E731
    lib(variant).rp_grad_cost_p(shape.encode(), p(pp), p(poly), 0 if poly is None else poly.size // 2,
                                occ.ctypes.data_as(C.POINTER(C.c_uint8)), X, Y, Z, p(lo), float(res), p(half), float(safety_hor),
                                poses.shape[0], p(poses), p(out))
    return out
