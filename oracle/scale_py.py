"""ctypes wrappers for the deformable-robot checkers — TEST INFRASTRUCTURE ONLY.

  * ScaledOracle: the oracle's scaled path (oracle/svsdf_oracle_scale.hpp via _build/libsvsdf_oracle_scale*.so), the checker of
    the scaled CUDA kernels; variant "default" (portable sin/cos, the strict build's bits) or "glibc".
  * RefScaled: the reference's own code with `useScale` on (_ref/libref_path_scaled_{glibc,portable}.so, only where the reference
    tree was present at build time), the RefPath of oracle/ref_py.py plus the schedule.
Schedules are 8 values: a_x, a_y, b_x, b_y, w_x, w_y, phi_x, phi_y.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import native, ref_py

_VARIANTS = {"default": "_build/libsvsdf_oracle_scale.so", "glibc": "_build/libsvsdf_oracle_scale_glibc.so"}
dp = C.POINTER(C.c_double)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _p(a):
    return a.ctypes.data_as(dp) if a is not None else None


def build() -> None:
    native.make("scale")


def build_ref() -> None:
    """The reference's own code with useScale on (needs the reference tree)."""
    native.make("ref_scaled")


def lib(variant: str = "default"):
    return native.load(_VARIANTS[variant], _declare, build)


def _declare(L):
    vp = C.c_void_p
    L.sorc_create.restype = vp
    L.sorc_create.argtypes = [C.c_char_p, dp, dp, C.c_int, C.c_double, C.c_double, C.c_int]
    L.sorc_create_mesh.restype = vp
    L.sorc_create_mesh.argtypes = [dp, dp, C.c_int, vp, C.c_int, C.c_double, C.c_double, C.c_int]
    L.sorc_destroy.argtypes = [vp]
    L.sorc_set_threads.argtypes = [vp, C.c_int]
    L.sorc_set_scale.argtypes = [vp, dp]
    L.sorc_scale_at.argtypes = [dp, C.c_double, dp, dp]
    L.sorc_set_points.argtypes = [vp, dp, C.c_int64, C.c_int]
    L.sorc_set_traj.argtypes = [vp, C.c_int, dp, dp]
    L.sorc_duration.restype = C.c_double
    L.sorc_duration.argtypes = [vp]
    L.sorc_traj_pos.argtypes = [vp, C.c_double, dp]
    L.sorc_traj_vel.argtypes = [vp, C.c_double, dp]
    L.sorc_sdf_at.restype = C.c_double
    L.sorc_sdf_at.argtypes = [vp, dp, C.c_double, C.c_int]
    L.sorc_gradient_descent.argtypes = [vp, dp, C.c_double, C.c_double, C.c_double, dp, dp]
    L.sorc_query_outer.argtypes = [vp, C.c_int64, dp, dp, dp, dp]
    L.sorc_query.argtypes = [vp, C.c_int64, dp, dp, dp, dp, C.POINTER(C.c_int)]
    L.sorc_cost_grad.restype = C.c_int64
    L.sorc_cost_grad.argtypes = [vp, C.c_int, dp, dp, dp, dp, dp, dp]


def scale_at(sched, t, variant="default"):
    """(S diagonal (sx, sy), St.inverse() diagonal (3,)) at time t, with the variant's sin."""
    s = _f64(sched).reshape(8)
    s2, inv3 = np.empty(2), np.empty(3)
    lib(variant).sorc_scale_at(_p(s), float(t), _p(s2), _p(inv3))
    return s2, inv3


class ScaledOracle:
    """The oracle's SweptVolumeManager + penalty loop for a deformable robot (schedule `sched`)."""

    def __init__(self, shape="star", sched=(1.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0), poly_params=(0.0, 0.0, 0.0), weight_p=60.0,
                 safety_hor=0.7, threads=1, polygon=None, mesh=None, variant="default"):
        self.L = lib(variant)
        pp = _f64(poly_params)
        if mesh is not None:  # (V, F): the triangle-mesh functor
            V = _f64(mesh[0]).reshape(-1, 3)
            F = np.ascontiguousarray(mesh[1], dtype=np.int32).reshape(-1, 3)
            self.h = self.L.sorc_create_mesh(_p(pp), _p(V), V.shape[0], F.ctypes.data_as(C.c_void_p), F.shape[0], weight_p,
                                             safety_hor, threads)
        else:
            poly = _f64(polygon).reshape(-1) if polygon is not None else None
            self.h = self.L.sorc_create(shape.encode(), _p(pp), _p(poly), 0 if poly is None else poly.size // 2, weight_p,
                                        safety_hor, threads)
        self.P = 0
        self.set_scale(sched)

    def __del__(self):
        try:
            if self.h:
                self.L.sorc_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def set_scale(self, sched):
        s = _f64(sched).reshape(8)
        self.L.sorc_set_scale(self.h, _p(s))

    def set_threads(self, n):
        self.L.sorc_set_threads(self.h, int(n))

    def set_points(self, pts):
        pts = _f64(pts)
        self.L.sorc_set_points(self.h, _p(pts), pts.shape[0], pts.shape[1])
        self.P = pts.shape[0]

    def set_traj(self, T, coeffs_colmajor):
        T = _f64(T)
        c = _f64(coeffs_colmajor).reshape(-1)
        self.L.sorc_set_traj(self.h, T.shape[0], _p(T), _p(c))

    def duration(self):
        return self.L.sorc_duration(self.h)

    def traj_pos(self, t):
        out = np.empty(3)
        self.L.sorc_traj_pos(self.h, float(t), _p(out))
        return out

    def traj_vel(self, t):
        out = np.empty(3)
        self.L.sorc_traj_vel(self.h, float(t), _p(out))
        return out

    def sdf_at(self, p, t, scaled=True):
        """getSDFAtTimeStamp at absolute time t: scaled (the descent's) or rigid (the seed scan's)."""
        p = _f64(p)
        return self.L.sorc_sdf_at(self.h, _p(p), float(t), int(bool(scaled)))

    def gradient_descent(self, p, tmin, tmax, x0):
        p = _f64(p)
        fx, x = C.c_double(), C.c_double()
        self.L.sorc_gradient_descent(self.h, _p(p), tmin, tmax, x0, C.cast(C.byref(fx), dp), C.cast(C.byref(x), dp))
        return fx.value, x.value

    def query_outer(self, pts):
        """The outer solve alone (choiceTInit rigid + the scaled descent): sdf, t*, body-frame gradient per point."""
        pts = _f64(pts).reshape(-1, 3)
        n = pts.shape[0]
        sdf, ts, g = np.empty(n), np.empty(n), np.empty((n, 3))
        self.L.sorc_query_outer(self.h, n, _p(pts), _p(sdf), _p(ts), _p(g))
        return sdf, ts, g

    def query(self, pts):
        pts = _f64(pts).reshape(-1, 3)
        n = pts.shape[0]
        sdf, ts, g = np.empty(n), np.empty(n), np.empty((n, 3))
        rounds = np.zeros(n, dtype=np.int32)
        self.L.sorc_query(self.h, n, _p(pts), _p(sdf), _p(ts), _p(g), rounds.ctypes.data_as(C.POINTER(C.c_int)))
        return sdf, ts, g, rounds

    def cost_grad(self, T, coeffs_colmajor, per_point=False):
        T = _f64(T)
        c = _f64(coeffs_colmajor).reshape(-1)
        N = T.shape[0]
        cost = C.c_double(0.0)
        gT, gC = np.zeros(N), np.zeros(18 * N)
        pp = np.empty((self.P, 7)) if per_point else None
        inside = self.L.sorc_cost_grad(self.h, N, _p(T), _p(c), C.cast(C.byref(cost), dp), _p(gT), _p(gC), _p(pp))
        return cost.value, gT, gC, pp, int(inside)


def ref_available() -> bool:
    return ref_py.available("scaled_glibc") and ref_py.available("scaled_portable")


class RefScaled(ref_py.RefPath):
    """The reference's own code with useScale on; variant "glibc" or "portable"."""

    def __init__(self, shape="star", sched=(1.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0), variant="glibc", **kw):
        super().__init__(shape, variant="scaled_" + variant, **kw)
        self.L.ref_scaled.restype = C.c_int
        assert self.L.ref_scaled() == 1
        self.L.ref_set_scale.argtypes = [C.c_void_p, dp]
        s = _f64(sched).reshape(8)
        self.L.ref_set_scale(self.h, _p(s))
