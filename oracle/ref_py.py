"""ctypes wrapper over oracle/_ref/libref_path_<variant>.so — the REFERENCE'S OWN SOURCE of the hot path, compiled where
it lies (oracle/ref_path_shim.cpp, oracle/ref_extract.py, oracle/ref_shim/).  TEST INFRASTRUCTURE ONLY.

The libraries exist only where /root/reference does (this container; they travel to the GPU box as built .so files, the
reference tree does not).  `RefPath` mirrors `oracle_py.Oracle` method for method so a test can drive both through the
same code and compare bit for bit; `tests/golden/make_ref_pin_golden.py` uses it to write the committed fixtures.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import native

VARIANTS = ("glibc", "portable", "glibc_r1", "glibc_r2")
dp = C.POINTER(C.c_double)
u8p = C.POINTER(C.c_uint8)


def _so(variant: str) -> str:
    return f"_ref/libref_path_{variant}.so"


def available(variant: str = "glibc") -> bool:
    return native.available(_so(variant))


def build() -> None:
    """The rigid path's pins and the mid end's (needs the reference tree)."""
    native.make("ref_path")


def lib(variant: str = "glibc"):
    return native.load(_so(variant), _declare)


def _declare(L):
    L.ref_variant.restype = C.c_char_p
    L.ref_redux_order.restype = C.c_int
    L.ref_shape_sdf.argtypes = [C.c_char_p, dp, dp, C.c_int, C.c_int64, dp, dp]
    L.ref_shape_grad1.argtypes = [C.c_char_p, dp, dp, C.c_int, C.c_int64, dp, dp]
    L.ref_shape_kernels.argtypes = [C.c_char_p, dp, C.c_int, C.c_int, C.c_double, C.c_double, dp, u8p, u8p]
    L.ref_smoothed_l1.argtypes = [C.c_int64, dp, C.c_double, dp, dp, u8p]
    L.ref_create.restype = C.c_void_p
    L.ref_create.argtypes = [C.c_char_p, dp, dp, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int]
    L.ref_destroy.argtypes = [C.c_void_p]
    L.ref_set_threads.argtypes = [C.c_void_p, C.c_int]
    L.ref_set_points.argtypes = [C.c_void_p, dp, C.c_int64, C.c_int]
    L.ref_set_traj.argtypes = [C.c_void_p, C.c_int, dp, dp]
    L.ref_traj_duration.restype = C.c_double
    L.ref_traj_duration.argtypes = [C.c_void_p]
    L.ref_traj_pos.argtypes = [C.c_void_p, C.c_double, dp]
    L.ref_traj_vel.argtypes = [C.c_void_p, C.c_double, dp]
    L.ref_locate_piece.restype = C.c_int
    L.ref_locate_piece.argtypes = [C.c_void_p, C.c_double, dp]
    L.ref_sdf_at.restype = C.c_double
    L.ref_sdf_at.argtypes = [C.c_void_p, dp, C.c_double]
    L.ref_sdf_dot_at.restype = C.c_double
    L.ref_sdf_dot_at.argtypes = [C.c_void_p, dp, C.c_double]
    L.ref_choice_t_init.restype = C.c_double
    L.ref_choice_t_init.argtypes = [C.c_void_p, dp, C.c_double]
    L.ref_gradient_descent.argtypes = [C.c_void_p, dp, C.c_double, C.c_double, C.c_double, dp, dp]
    L.ref_query_outer.argtypes = [C.c_void_p, C.c_int64, dp, dp, dp, dp]
    L.ref_query.argtypes = [C.c_void_p, C.c_int64, dp, dp, dp, dp]
    L.ref_cost_grad.argtypes = [C.c_void_p, C.c_int, dp, dp, dp, dp, dp]
    L.ref_set_conditions.argtypes = [C.c_void_p, dp, dp, C.c_int]
    L.ref_evaluate.restype = C.c_double
    L.ref_evaluate.argtypes = [C.c_void_p, dp, dp, C.c_int]
    L.ref_last_costs.argtypes = [C.c_void_p, dp]
    L.ref_minco_forward.argtypes = [C.c_void_p, dp, dp, dp, dp, dp, dp]
    L.ref_minco_propagate.argtypes = [C.c_void_p, dp, dp, dp, dp]
    L.ref_forward_T.argtypes = [C.c_int, dp, dp]
    L.ref_backward_T.argtypes = [C.c_int, dp, dp]


def _p(a):
    return a.ctypes.data_as(dp) if a is not None else None


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def shape_sdf(name, rel, poly_params=(0.0, 0.0, 0.0), polygon=None, variant="glibc"):
    rel = _f64(rel).reshape(-1, 3)
    out = np.empty(rel.shape[0])
    pp = _f64(poly_params)
    poly = _f64(polygon).reshape(-1) if polygon is not None else None
    lib(variant).ref_shape_sdf(name.encode(), _p(pp), _p(poly), 0 if poly is None else poly.size // 2, rel.shape[0], _p(rel), _p(out))
    return out


def shape_grad1(name, rel, poly_params=(0.0, 0.0, 0.0), polygon=None, variant="glibc"):
    rel = _f64(rel).reshape(-1, 3)
    out = np.empty((rel.shape[0], 3))
    pp = _f64(poly_params)
    poly = _f64(polygon).reshape(-1) if polygon is not None else None
    lib(variant).ref_shape_grad1(name.encode(), _p(pp), _p(poly), 0 if poly is None else poly.size // 2, rel.shape[0], _p(rel), _p(out))
    return out


def shape_kernels(name, kernel_size=17, kernel_count=18, res=1.0, safeh=0.0, poly_params=(0.0, 0.0, 0.0), variant="glibc"):
    """BasicShape::initShape: (yaw[K], cells[K, ks, ks] uint8, bytes[K, ks, ceil(ks/8)] uint8)."""
    ks, K = int(kernel_size), int(kernel_count)
    yaw = np.empty(K)
    cells = np.zeros((K, ks, ks), dtype=np.uint8)
    byt = np.zeros((K, ks, (ks + 7) // 8), dtype=np.uint8)
    pp = _f64(poly_params)
    lib(variant).ref_shape_kernels(name.encode(), _p(pp), ks, K, float(res), float(safeh), _p(yaw), cells.ctypes.data_as(u8p),
                                   byt.ctypes.data_as(u8p))
    return yaw, cells, byt


def smoothed_l1(x, mu=0.01, variant="glibc"):
    x = _f64(x).reshape(-1)
    f, df = np.empty_like(x), np.empty_like(x)
    ret = np.zeros(x.size, dtype=np.uint8)
    lib(variant).ref_smoothed_l1(x.size, _p(x), float(mu), _p(f), _p(df), ret.ctypes.data_as(u8p))
    return ret.astype(bool), f, df


def forward_T(tau, variant="glibc"):
    tau = _f64(tau)
    T = np.empty_like(tau)
    lib(variant).ref_forward_T(tau.size, _p(tau), _p(T))
    return T


def backward_T(T, variant="glibc"):
    T = _f64(T)
    tau = np.empty_like(T)
    lib(variant).ref_backward_T(T.size, _p(T), _p(tau))
    return tau


class RefPath:
    """The reference's SweptVolumeManager + TrajOptimizer (its own code) for one shape; mirrors oracle_py.Oracle."""

    def __init__(self, shape="star", poly_params=(0.0, 0.0, 0.0), weight_p=60.0, safety_hor=0.7, rho=3.8, threads=1, polygon=None,
                 variant="glibc"):
        pp = _f64(poly_params)
        poly = _f64(polygon).reshape(-1) if polygon is not None else None
        self.L = lib(variant)
        self.N = 0
        self.P = 0
        self.h = self.L.ref_create(shape.encode(), _p(pp), _p(poly), 0 if poly is None else poly.size // 2, weight_p, safety_hor, rho, threads)

    def __del__(self):
        try:
            if self.h:
                self.L.ref_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def set_threads(self, n):
        self.L.ref_set_threads(self.h, int(n))

    def set_points(self, pts):
        pts = _f64(pts)
        self.L.ref_set_points(self.h, _p(pts), pts.shape[0], pts.shape[1])
        self.P = pts.shape[0]

    def set_traj(self, T, coeffs_colmajor):
        T = _f64(T)
        c = _f64(coeffs_colmajor).reshape(-1)
        self.N = T.shape[0]
        self.L.ref_set_traj(self.h, self.N, _p(T), _p(c))

    def duration(self):
        return self.L.ref_traj_duration(self.h)

    def traj_pos(self, t):
        out = np.empty(3)
        self.L.ref_traj_pos(self.h, float(t), _p(out))
        return out

    def traj_vel(self, t):
        out = np.empty(3)
        self.L.ref_traj_vel(self.h, float(t), _p(out))
        return out

    def locate_piece(self, t):
        tl = C.c_double()
        i = self.L.ref_locate_piece(self.h, float(t), C.cast(C.byref(tl), dp))
        return i, tl.value

    def sdf_at(self, p, t):
        p = _f64(p)
        return self.L.ref_sdf_at(self.h, _p(p), float(t))

    def sdf_dot_at(self, p, t):
        p = _f64(p)
        return self.L.ref_sdf_dot_at(self.h, _p(p), float(t))

    def choice_t_init(self, p, dt=0.15):
        p = _f64(p)
        return self.L.ref_choice_t_init(self.h, _p(p), dt)

    def gradient_descent(self, p, tmin, tmax, x0):
        p = _f64(p)
        fx = C.c_double()
        x = C.c_double()
        self.L.ref_gradient_descent(self.h, _p(p), tmin, tmax, x0, C.cast(C.byref(fx), dp), C.cast(C.byref(x), dp))
        return fx.value, x.value

    def query_outer(self, pts):
        pts = _f64(pts).reshape(-1, 3)
        n = pts.shape[0]
        sdf, ts, g = np.empty(n), np.empty(n), np.empty((n, 3))
        self.L.ref_query_outer(self.h, n, _p(pts), _p(sdf), _p(ts), _p(g))
        return sdf, ts, g

    def query(self, pts):
        pts = _f64(pts).reshape(-1, 3)
        n = pts.shape[0]
        sdf, ts, g = np.empty(n), np.empty(n), np.empty((n, 3))
        self.L.ref_query(self.h, n, _p(pts), _p(sdf), _p(ts), _p(g))
        return sdf, ts, g

    def cost_grad(self, T, coeffs_colmajor, cost0=0.0, gradT0=None, gradC0=None):
        T = _f64(T)
        c = _f64(coeffs_colmajor).reshape(-1)
        N = T.shape[0]
        cost = C.c_double(cost0)
        gT = np.zeros(N) if gradT0 is None else _f64(gradT0).copy()
        gC = np.zeros(18 * N) if gradC0 is None else _f64(gradC0).reshape(-1).copy()
        self.L.ref_cost_grad(self.h, N, _p(T), _p(c), C.cast(C.byref(cost), dp), _p(gT), _p(gC))
        return cost.value, gT, gC

    def set_conditions(self, init_s, final_s, N):
        i_s = _f64(np.asarray(init_s).T).reshape(-1)
        f_s = _f64(np.asarray(final_s).T).reshape(-1)
        self.N = N
        self.L.ref_set_conditions(self.h, _p(i_s), _p(f_s), N)

    def evaluate(self, x):
        x = _f64(x)
        g = np.empty_like(x)
        f = self.L.ref_evaluate(self.h, _p(x), _p(g), x.shape[0])
        return f, g

    def last_costs(self):
        out = np.empty(3)
        self.L.ref_last_costs(self.h, _p(out))
        return out

    def minco_forward(self, q, T):
        """q: 3 x (N-1); returns b (18N, column-major), energy, dE/dc (18N), dE/dT (N) from the reference's MINCO_S3NU."""
        N = self.N
        qf = _f64(np.asarray(q).T).reshape(-1)  # column i = waypoint i -> (x, y, yaw) contiguous
        T = _f64(T)
        b, gdC, gdT = np.empty(18 * N), np.empty(18 * N), np.empty(N)
        e = C.c_double()
        self.L.ref_minco_forward(self.h, _p(qf), _p(T), _p(b), C.cast(C.byref(e), dp), _p(gdC), _p(gdT))
        return b, e.value, gdC, gdT

    def minco_propagate(self, gdC, gdT):
        N = self.N
        gdC, gdT = _f64(gdC).reshape(-1), _f64(gdT)
        gP, gT = np.empty(3 * (N - 1)), np.empty(N)
        self.L.ref_minco_propagate(self.h, _p(gdC), _p(gdT), _p(gP), _p(gT))
        return gP.reshape(N - 1, 3).T.copy(), gT


# ---- mid end: the reference's OriTraj (oracle/ref_mid_shim.cpp -> oracle/_ref/libref_mid.so) ----
def mid_available() -> bool:
    return native.available("_ref/libref_mid.so")


def _mid_lib():
    return native.load("_ref/libref_mid.so", lambda L: None)


def mid_cost(cfg, N, init_cm, final_cm, Q_cm, rot_cm, x):
    """OriTraj::costFunction of the reference.  cfg: a ctypes struct with svsdf_mid_config's layout; arrays flat, column-major as
    the C ABI takes them."""
    dp = C.POINTER(C.c_double)
    f = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    x = f(x)
    g = np.zeros_like(x)
    cost = C.c_double()
    a = [f(init_cm), f(final_cm), f(Q_cm), f(rot_cm)]
    _mid_lib().ref_mid_cost(C.byref(cfg), C.c_int(N), *[v.ctypes.data_as(dp) for v in a], x.ctypes.data_as(dp), C.byref(cost), g.ctypes.data_as(dp))
    return cost.value, g


def mid_get_ori_traj(cfg, N, init_cm, final_cm, Q_cm, T_init, rot_cm):
    """OriTraj::getOriTraj of the reference with its own patched L-BFGS: (ok, opt_x, T, coeffs [6N, 3], iterations)."""
    dp = C.POINTER(C.c_double)
    f = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    a = [f(init_cm), f(final_cm), f(Q_cm), f(T_init), f(rot_cm)]
    x = np.zeros(N + 3 * (N - 1))
    T = np.zeros(N)
    co = np.zeros(18 * N)
    it = C.c_int()
    ok = _mid_lib().ref_mid_get_ori_traj(C.byref(cfg), C.c_int(N), *[v.ctypes.data_as(dp) for v in a], x.ctypes.data_as(dp), T.ctypes.data_as(dp),
                                         co.ctypes.data_as(dp), C.byref(it))
    return bool(ok), x, T, co.reshape(3, 6 * N).T.copy(), it.value
