"""ctypes wrapper of the swept-volume contour checker (oracle/swept_oracle.hpp) — TEST INFRASTRUCTURE ONLY.

swept_contour(field, i0, j0, h, iso) contours a dense field (ny x nx, NaN = not evaluated) by the svsdf_swept_contour contract and
returns a SimpleNamespace with vertices (V x 2), segments (S x 2), triangles (F x 3) and clipped.
"""
from __future__ import annotations

import ctypes as C
import types

import numpy as np

from . import native

_SO = "_build/libsvsdf_oracle_swept.so"


def build() -> None:
    native.make("swept")


def lib():
    return native.load(_SO, _declare, build)


def _declare(L):
    L.sw_contour.restype = C.c_void_p
    L.sw_contour.argtypes = [C.POINTER(C.c_double), C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_double, C.c_double,
                             C.POINTER(C.c_int64)]
    L.sw_copy.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.sw_free.argtypes = [C.c_void_p]


def swept_contour(field, i0, j0, h, iso):
    f = np.ascontiguousarray(field, dtype=np.float64)
    assert f.ndim == 2 and f.shape[0] >= 2 and f.shape[1] >= 2, f.shape
    ny, nx = f.shape
    L = lib()
    sizes = (C.c_int64 * 4)()
    hd = L.sw_contour(f.ctypes.data_as(C.POINTER(C.c_double)), int(i0), int(j0), nx, ny, float(h), float(iso), sizes)
    try:
        V, S, F = sizes[0], sizes[1], sizes[2]
        v = np.empty((V, 2))
        s = np.empty((S, 2), dtype=np.int32)
        t = np.empty((F, 3), dtype=np.int32)
        L.sw_copy(hd, v.ctypes.data, s.ctypes.data, t.ctypes.data)
    finally:
        L.sw_free(hd)
    return types.SimpleNamespace(vertices=v, segments=s, triangles=t, clipped=int(sizes[3]))
