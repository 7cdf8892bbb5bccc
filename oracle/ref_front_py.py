"""ctypes wrapper over oracle/_ref/libref_front_<variant>.so — the REFERENCE'S OWN SOURCE of the A* front end (node test and
search), compiled where it lies (oracle/ref_front_shim.cpp, oracle/ref_extract_front.py).  TEST INFRASTRUCTURE ONLY.

The libraries exist only where the reference tree does; the tests that compare against them read the recorded outputs in
tests/golden/ref_pin_front.npz elsewhere (tests/golden/make_front_golden.py writes it).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import native

VARIANTS = ("glibc", "portable")
dp = C.POINTER(C.c_double)
u8p = C.POINTER(C.c_uint8)
i32p = C.POINTER(C.c_int32)


def available(variant: str = "portable") -> bool:
    return native.available(f"_ref/libref_front_{variant}.so")


def lib(variant: str = "portable"):
    return native.load(f"_ref/libref_front_{variant}.so", lambda L: _declare(L, variant))


def _declare(L, variant):
    L.rf_variant.restype = C.c_char_p
    L.rf_create.restype = C.c_void_p
    L.rf_create.argtypes = [C.c_char_p, dp, C.c_int, C.c_int, C.c_double, C.c_double, u8p, C.c_int, C.c_int, C.c_double, C.c_double]
    L.rf_destroy.argtypes = [C.c_void_p]
    L.rf_map_kernel.restype = C.c_int
    L.rf_map_kernel.argtypes = [C.c_void_p, u8p]
    L.rf_kernels.argtypes = [C.c_void_p, dp, u8p, u8p]
    L.rf_kernel_conv.argtypes = [C.c_void_p, C.c_int, C.c_int64, i32p, u8p]
    L.rf_check_kernel_value.argtypes = [C.c_void_p, C.c_int64, dp, i32p, u8p, dp]
    L.rf_points_in_aabb.restype = C.c_int64
    L.rf_points_in_aabb.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_double, dp, C.c_int64]
    L.rf_expand.argtypes = [C.c_void_p, C.c_int64, i32p, dp, u8p, dp, u8p]
    L.rf_astar.argtypes = [C.c_void_p, C.c_int, dp, dp, C.c_int, dp, i32p, i32p, u8p]
    assert L.rf_variant().decode() == variant


def _p(a, t):
    return a.ctypes.data_as(t)


class RefFront:
    """One reference front end: the shape's kernels (ks, K, res, safeh) and the map occ [X, Y] at `origin`, cell size res."""

    def __init__(self, name, occ, origin, res, ks, K, safeh=0.0, poly_params=(0.0, 0.0, 0.0), variant="portable"):
        self.L = lib(variant)
        self.occ = np.ascontiguousarray(occ, dtype=np.uint8)
        self.X, self.Y = self.occ.shape
        self.ks, self.K = int(ks), int(K)
        pp = np.ascontiguousarray(poly_params, dtype=np.float64)
        self.h = self.L.rf_create(name.encode(), _p(pp, dp), self.ks, self.K, float(res), float(safeh), _p(self.occ, u8p), self.X, self.Y,
                                  float(origin[0]), float(origin[1]))
        if not self.h:
            raise ValueError(name)

    def close(self):
        if self.h:
            self.L.rf_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def map_kernel(self):
        n = self.L.rf_map_kernel(self.h, None)
        out = np.zeros(n, dtype=np.uint8)
        self.L.rf_map_kernel(self.h, _p(out, u8p))
        return out

    def kernels(self):
        bpr = (self.ks + 7) // 8
        yaw = np.empty(self.K)
        cells = np.zeros((self.K, self.ks, self.ks), dtype=np.uint8)
        byt = np.zeros((self.K, self.ks, bpr), dtype=np.uint8)
        self.L.rf_kernels(self.h, _p(yaw, dp), _p(cells, u8p), _p(byt, u8p))
        return yaw, cells.astype(bool), byt

    def cspace(self, byte_variant=True):
        """kernelConv over every (yaw kernel, cell): bool [K, X, Y], True = free."""
        k, i, j = np.meshgrid(np.arange(self.K), np.arange(self.X), np.arange(self.Y), indexing="ij")
        kij = np.ascontiguousarray(np.stack([k.ravel(), i.ravel(), j.ravel()], axis=1), dtype=np.int32)
        out = np.zeros(kij.shape[0], dtype=np.uint8)
        self.L.rf_kernel_conv(self.h, 1 if byte_variant else 0, kij.shape[0], _p(kij, i32p), _p(out, u8p))
        return out.reshape(self.K, self.X, self.Y).astype(bool)

    def check_kernel_value(self, father_yaw, ind_xy):
        fy = np.ascontiguousarray(father_yaw, dtype=np.float64).reshape(-1)
        ij = np.ascontiguousarray(ind_xy, dtype=np.int32).reshape(-1, 2)
        ok = np.zeros(fy.size, dtype=np.uint8)
        cy = np.empty(fy.size)
        self.L.rf_check_kernel_value(self.h, fy.size, _p(fy, dp), _p(ij, i32p), _p(ok, u8p), _p(cy, dp))
        return ok.astype(bool), cy

    def points_in_aabb(self, centre, half):
        cap = self.X * self.Y
        xy = np.empty((max(cap, 1), 2))
        m = self.L.rf_points_in_aabb(self.h, float(centre[0]), float(centre[1]), float(half), float(half), _p(xy, dp), cap)
        return xy[:m].copy()

    def expand(self, node_ij, node_yaw):
        """(ok [n, 9] bool, child_yaw [n, 9], parts [n, 9]) — see rf_expand."""
        ij = np.ascontiguousarray(node_ij, dtype=np.int32).reshape(-1, 2)
        fy = np.ascontiguousarray(node_yaw, dtype=np.float64).reshape(-1)
        n = fy.size
        ok = np.zeros((n, 9), dtype=np.uint8)
        cy = np.zeros((n, 9))
        parts = np.zeros((n, 9), dtype=np.uint8)
        self.L.rf_expand(self.h, n, _p(ij, i32p), _p(fy, dp), _p(ok, u8p), _p(cy, dp), _p(parts, u8p))
        return ok.astype(bool), cy, parts

    def astar(self, start_xy, goal_xy, max_path=4096):
        """(paths: list of [len, 3] or None, expansions [n], found [n])."""
        st = np.ascontiguousarray(start_xy, dtype=np.float64).reshape(-1, 2)
        go = np.ascontiguousarray(goal_xy, dtype=np.float64).reshape(-1, 2)
        n = st.shape[0]
        path = np.zeros((n, max_path, 3))
        ln = np.zeros(n, dtype=np.int32)
        ex = np.zeros(n, dtype=np.int32)
        found = np.zeros(n, dtype=np.uint8)
        self.L.rf_astar(self.h, n, _p(st, dp), _p(go, dp), max_path, _p(path, dp), _p(ln, i32p), _p(ex, i32p), _p(found, u8p))
        return [path[q, : ln[q]].copy() if ln[q] else None for q in range(n)], ex, found.astype(bool)
