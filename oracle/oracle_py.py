"""ctypes wrapper over oracle/_build/libsvsdf_oracle.so — TEST INFRASTRUCTURE ONLY.

Importers allowed: tests/, __graft_entry__.smoke(), bench.py (cpu_baseline / --impl reference legs).
The product package (implicit_svsdf_planner_b200/) must never import this module.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import native

_VARIANTS = {"default": "_build/libsvsdf_oracle.so", "fma": "_build/libsvsdf_oracle_fma.so", "glibc": "_build/libsvsdf_oracle_glibc.so"}

dp = C.POINTER(C.c_double)


def build() -> str:
    native.make("oracle")
    return native.path(_VARIANTS["default"])


def lib(variant: str = "default"):
    """variant "default": portable (fdlibm) sin/cos, no FMA contraction — bit-compatible with the strict CUDA build;
    "glibc": std::sin/std::cos, no contraction (the reference's x86-64 behaviour; timed as the CPU baseline);
    "fma": glibc sin/cos with -ffp-contract=fast -mfma (what the same source does on FMA targets)."""
    return native.load(_VARIANTS[variant], _declare, build)


def _declare(L):
    L.orc_sincos.argtypes = [C.c_int64, dp, dp, dp]
    L.orc_atan2.argtypes = [C.c_int64, dp, dp, dp]
    L.orc_create.restype = C.c_void_p
    L.orc_create.argtypes = [C.c_char_p, dp, dp, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int]
    L.orc_destroy.argtypes = [C.c_void_p]
    L.orc_set_threads.argtypes = [C.c_void_p, C.c_int]
    L.orc_set_points.argtypes = [C.c_void_p, dp, C.c_int64, C.c_int]
    L.orc_set_traj.argtypes = [C.c_void_p, C.c_int, dp, dp]
    L.orc_traj_duration.restype = C.c_double
    L.orc_traj_duration.argtypes = [C.c_void_p]
    L.orc_traj_pos.argtypes = [C.c_void_p, C.c_double, dp]
    L.orc_traj_vel.argtypes = [C.c_void_p, C.c_double, dp]
    L.orc_sdf_at.restype = C.c_double
    L.orc_sdf_at.argtypes = [C.c_void_p, dp, C.c_double]
    L.orc_choice_t_init.restype = C.c_double
    L.orc_choice_t_init.argtypes = [C.c_void_p, dp, C.c_double]
    L.orc_gradient_descent.argtypes = [C.c_void_p, dp, C.c_double, C.c_double, C.c_double, dp, dp]
    L.orc_count_evals.argtypes = [C.c_void_p, C.c_int]
    L.orc_eval_count.restype = C.c_uint64
    L.orc_eval_count.argtypes = [C.c_void_p]
    L.orc_query_outer.argtypes = [C.c_void_p, C.c_int64, dp, dp, dp, dp]
    L.orc_query.argtypes = [C.c_void_p, C.c_int64, dp, dp, dp, dp, C.POINTER(C.c_int)]
    L.orc_cost_grad.restype = C.c_int64
    L.orc_cost_grad.argtypes = [C.c_void_p, C.c_int, dp, dp, dp, dp, dp, dp]
    L.orc_time_cost_grad.restype = C.c_double
    L.orc_time_cost_grad.argtypes = [C.c_void_p, C.c_int, dp, dp, C.c_int, C.c_int, dp]
    L.orc_shape_sdf.argtypes = [C.c_char_p, dp, dp, C.c_int, C.c_int64, dp, dp]
    L.orc_shape_grad1.argtypes = [C.c_char_p, dp, dp, C.c_int, C.c_int64, dp, dp]
    L.orc_minco_forward.argtypes = [dp, dp, C.c_int, dp, dp, dp, dp, dp, dp]
    L.orc_minco_propagate.argtypes = [dp, dp, C.c_int, dp, dp, dp, dp, dp, dp]
    L.orc_forward_T.argtypes = [C.c_int, dp, dp]
    L.orc_backward_T.argtypes = [C.c_int, dp, dp]
    L.orc_set_conditions.argtypes = [C.c_void_p, dp, dp, C.c_int]
    L.orc_evaluate.restype = C.c_double
    L.orc_evaluate.argtypes = [C.c_void_p, dp, dp, C.c_int]
    L.orc_last_costs.argtypes = [C.c_void_p, dp]
    L.orc_get_coeffs.argtypes = [C.c_void_p, dp, dp]
    L.orc_lbfgs.restype = C.c_int
    L.orc_lbfgs.argtypes = [C.c_void_p, dp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_double, dp]
    L.orc_mesh_eval.argtypes = [dp, dp, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int64, dp, dp]
    L.orc_create_mesh.restype = C.c_void_p
    L.orc_create_mesh.argtypes = [dp, dp, C.c_int, C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int]
    u8 = C.POINTER(C.c_uint8)
    L.orc_shape_kernels.argtypes = [C.c_char_p, dp, C.c_int, C.c_int, C.c_double, C.c_double, dp, u8, u8]
    L.orc_cspace.argtypes = [C.c_char_p, dp, C.c_int, C.c_int, C.c_double, C.c_double, u8, C.c_int, C.c_int, C.c_int, u8]
    L.orc_check_kernel_value.argtypes = [C.c_char_p, dp, C.c_int, C.c_int, C.c_double, C.c_double, u8, C.c_int, C.c_int, C.c_int64, dp,
                                         C.POINTER(C.c_int), u8, dp]
    L.orc_expand_nodes.argtypes = [C.c_char_p, dp, C.c_int, C.c_int, C.c_double, C.c_double, u8, C.c_int, C.c_int, C.c_double, C.c_double,
                                   C.c_double, C.c_int64, C.POINTER(C.c_int), dp, u8, dp, u8]
    L.orc_astar.argtypes = [C.c_char_p, dp, C.c_int, C.c_int, C.c_double, u8, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, dp,
                            dp, C.c_int, dp, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.orc_points_in_aabb.restype = C.c_int64
    L.orc_points_in_aabb.argtypes = [u8, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double,
                                     C.c_double, dp, C.c_int64]
    L.orc_max_threads.restype = C.c_int
    L.orc_num_procs.restype = C.c_int


def _p(a):
    return a.ctypes.data_as(dp) if a is not None else None


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def shape_sdf(name, rel, poly_params=(0.0, 0.0, 0.0), polygon=None):
    rel = _f64(rel).reshape(-1, 3)
    out = np.empty(rel.shape[0])
    pp = _f64(poly_params)
    poly = _f64(polygon).reshape(-1) if polygon is not None else None
    lib().orc_shape_sdf(name.encode(), _p(pp), _p(poly), 0 if poly is None else poly.size // 2, rel.shape[0], _p(rel), _p(out))
    return out


def shape_grad1(name, rel, poly_params=(0.0, 0.0, 0.0), polygon=None):
    rel = _f64(rel).reshape(-1, 3)
    out = np.empty((rel.shape[0], 3))
    pp = _f64(poly_params)
    poly = _f64(polygon).reshape(-1) if polygon is not None else None
    lib().orc_shape_grad1(name.encode(), _p(pp), _p(poly), 0 if poly is None else poly.size // 2, rel.shape[0], _p(rel), _p(out))
    return out


def _mesh_args(mesh):
    V = _f64(mesh[0]).reshape(-1, 3)
    F = np.ascontiguousarray(mesh[1], dtype=np.int32).reshape(-1, 3)
    return V, F


def mesh_eval(mesh, rel, what="sdf", poly_params=(0.0, 0.0, 0.0)):
    """BasicShape::getonlySDF_igl restatement over body-frame points; what in sdf | winding | sqr_distance | grad1 (as the
    reference computes them: float winding-number hierarchy) | winding_exact | sdf_exact (exact double sum over the faces)."""
    V, F = _mesh_args(mesh)
    rel = _f64(rel).reshape(-1, 3)
    code = {"sdf": 0, "winding": 1, "sqr_distance": 2, "grad1": 3, "winding_exact": 4, "sdf_exact": 5}[what]
    out = np.empty((rel.shape[0], 3)) if code == 3 else np.empty(rel.shape[0])
    pp = _f64(poly_params)
    lib().orc_mesh_eval(_p(pp), _p(V), V.shape[0], F.ctypes.data_as(C.c_void_p), F.shape[0], code, rel.shape[0], _p(rel), _p(out))
    return out


def atan2f_pair(y, x):
    """(pinned fdlibm atan2f, C library atan2f) on float32 arrays."""
    y = np.ascontiguousarray(y, dtype=np.float32)
    x = np.ascontiguousarray(x, dtype=np.float32)
    a, b = np.empty_like(y), np.empty_like(y)
    fp = C.POINTER(C.c_float)
    lib().orc_atan2f_pair(C.c_int64(y.size), y.ctypes.data_as(fp), x.ctypes.data_as(fp), a.ctypes.data_as(fp), b.ctypes.data_as(fp))
    return a, b


def _u8p(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint8))


def shape_kernels(name, kernel_size=17, kernel_count=18, res=1.0, safeh=0.0, poly_params=(0.0, 0.0, 0.0)):
    """BasicShape::initShape: (yaw [K], bool kernels [K, ks, ks], byte kernels [K, ks, ceil(ks / 8)])."""
    pp = _f64(poly_params)
    bpr = (kernel_size + 7) // 8
    yaw = np.empty(kernel_count)
    cells = np.zeros((kernel_count, kernel_size, kernel_size), dtype=np.uint8)
    byt = np.zeros((kernel_count, kernel_size, bpr), dtype=np.uint8)
    lib().orc_shape_kernels(name.encode(), _p(pp), kernel_size, kernel_count, res, safeh, _p(yaw), _u8p(cells), _u8p(byt))
    return yaw, cells.astype(bool), byt


def cspace(name, occ, kernel_size=17, kernel_count=18, res=1.0, safeh=0.0, variant="byte", poly_params=(0.0, 0.0, 0.0)):
    """kernelConv over every (yaw kernel, cell): bool array [K, X, Y], True = the shape kernel meets no occupied cell."""
    occ = np.ascontiguousarray(occ, dtype=np.uint8)
    X, Y = occ.shape
    pp = _f64(poly_params)
    out = np.zeros((kernel_count, X, Y), dtype=np.uint8)
    lib().orc_cspace(name.encode(), _p(pp), kernel_size, kernel_count, res, safeh, _u8p(occ), X, Y, 1 if variant == "byte" else 0, _u8p(out))
    return out.astype(bool)


def check_kernel_value(name, occ, father_yaw, ind_xy, kernel_size=17, kernel_count=18, res=1.0, safeh=0.0, poly_params=(0.0, 0.0, 0.0)):
    """SweptVolumeManager::checkKernelValue for a batch: (ok [n] bool, child_yaw [n])."""
    occ = np.ascontiguousarray(occ, dtype=np.uint8)
    X, Y = occ.shape
    pp = _f64(poly_params)
    fy = _f64(father_yaw)
    ind = np.ascontiguousarray(ind_xy, dtype=np.int32).reshape(-1, 2)
    ok = np.zeros(fy.shape[0], dtype=np.uint8)
    cy = np.empty(fy.shape[0])
    lib().orc_check_kernel_value(name.encode(), _p(pp), kernel_size, kernel_count, res, safeh, _u8p(occ), X, Y, fy.shape[0], _p(fy),
                                 ind.ctypes.data_as(C.POINTER(C.c_int)), _u8p(ok), _p(cy))
    return ok.astype(bool), cy


def expand_nodes(name, occ, node_ij, node_yaw, origin=(0.0, 0.0), map_res=1.0, kernel_size=17, kernel_count=18, safeh=0.0,
                 poly_params=(0.0, 0.0, 0.0)):
    """The neighbour loop of the A* `process` step for n nodes: (ok [n, 9] bool, child_yaw [n, 9], parts [n, 9] bit mask:
    1 valid and free, 2 kernel test, 4 sub-swept-volume test).  The shape kernels use the map resolution as cell size."""
    occ = np.ascontiguousarray(occ, dtype=np.uint8)
    X, Y = occ.shape
    pp = _f64(poly_params)
    ij = np.ascontiguousarray(node_ij, dtype=np.int32).reshape(-1, 2)
    fy = _f64(node_yaw).reshape(-1)
    n = fy.size
    ok = np.zeros((n, 9), dtype=np.uint8)
    cy = np.zeros((n, 9))
    parts = np.zeros((n, 9), dtype=np.uint8)
    lib().orc_expand_nodes(name.encode(), _p(pp), kernel_size, kernel_count, float(map_res), safeh, _u8p(occ), X, Y, float(origin[0]),
                           float(origin[1]), float(map_res), n, ij.ctypes.data_as(C.POINTER(C.c_int)), _p(fy), _u8p(ok), _p(cy), _u8p(parts))
    return ok.astype(bool), cy, parts


def points_in_aabb(occ, centre, half, origin=(0.0, 0.0), map_res=1.0):
    """PCSmapManager::getPointsInAABB2D: the occupied cell centres [m, 2] in the box of half size `half` around `centre`."""
    occ = np.ascontiguousarray(occ, dtype=np.uint8)
    X, Y = occ.shape
    cap = X * Y
    xy = np.empty((max(cap, 1), 2))
    m = lib().orc_points_in_aabb(_u8p(occ), X, Y, float(origin[0]), float(origin[1]), float(map_res), float(centre[0]), float(centre[1]),
                                 float(half), float(half), _p(xy), cap)
    return xy[:m].copy()


def astar(name, occ, start_xy, goal_xy, origin=(0.0, 0.0), map_res=1.0, kernel_size=17, kernel_count=18, safeh=0.0, max_path=1024,
          poly_params=(0.0, 0.0, 0.0)):
    """AstarPathSearcher::AstarPathSearch + getPath for n start/goal pairs: (list of paths [len, 3] (x, y, yaw) or None, expansions [n])."""
    occ = np.ascontiguousarray(occ, dtype=np.uint8)
    X, Y = occ.shape
    pp = _f64(poly_params)
    st = _f64(start_xy).reshape(-1, 2)
    go = _f64(goal_xy).reshape(-1, 2)
    n = st.shape[0]
    path = np.zeros((n, max_path, 3))
    ln = np.zeros(n, dtype=np.int32)
    ex = np.zeros(n, dtype=np.int32)
    lib().orc_astar(name.encode(), _p(pp), kernel_size, kernel_count, safeh, _u8p(occ), X, Y, float(origin[0]), float(origin[1]), float(map_res), n,
                    _p(st), _p(go), max_path, _p(path), ln.ctypes.data_as(C.POINTER(C.c_int)), ex.ctypes.data_as(C.POINTER(C.c_int)))
    return [path[q, : ln[q]].copy() if ln[q] else None for q in range(n)], ex


def minco_forward(init_s, final_s, q, T):
    """init_s/final_s: 3x3 numpy [dim, derivative]; q: 3x(N-1); returns b (6N x 3), energy, gdC (6N x 3), gdT."""
    N = int(T.shape[0])
    i_s = _f64(np.asarray(init_s).T).reshape(-1)  # column-major 3x3
    f_s = _f64(np.asarray(final_s).T).reshape(-1)
    qq = _f64(np.asarray(q).T).reshape(-1)  # column-major 3x(N-1)
    TT = _f64(T)
    b = np.empty(18 * N)
    gdC = np.empty(18 * N)
    gdT = np.empty(N)
    e = C.c_double()
    lib().orc_minco_forward(_p(i_s), _p(f_s), N, _p(qq), _p(TT), _p(b), C.cast(C.byref(e), dp), _p(gdC), _p(gdT))
    return b.reshape(3, 6 * N).T.copy(), e.value, gdC.reshape(3, 6 * N).T.copy(), gdT


def minco_propagate(init_s, final_s, q, T, gdC, gdT):
    N = int(T.shape[0])
    i_s = _f64(np.asarray(init_s).T).reshape(-1)
    f_s = _f64(np.asarray(final_s).T).reshape(-1)
    qq = _f64(np.asarray(q).T).reshape(-1)
    TT = _f64(T)
    gc = _f64(np.asarray(gdC).T).reshape(-1)
    gt = _f64(gdT)
    gq = np.empty(3 * (N - 1))
    gT = np.empty(N)
    lib().orc_minco_propagate(_p(i_s), _p(f_s), N, _p(qq), _p(TT), _p(gc), _p(gt), _p(gq), _p(gT))
    return gq.reshape(N - 1, 3).T.copy(), gT


class Oracle:
    """Handle on the CPU restatement of TrajOptimizer + SweptVolumeManager for one shape."""

    def __init__(self, shape="star", poly_params=(0.0, 0.0, 0.0), weight_p=60.0, safety_hor=0.7, rho=3.8, threads=1, polygon=None,
                 variant="default", mesh=None):
        pp = _f64(poly_params)
        poly = _f64(polygon).reshape(-1) if polygon is not None else None
        self.L = lib(variant)
        self.N = 0
        if mesh is not None:  # (V, F): the triangle-mesh functor (getonlySDF_igl) instead of a registry shape
            V, F = _mesh_args(mesh)
            self.h = self.L.orc_create_mesh(_p(pp), _p(V), V.shape[0], F.ctypes.data_as(C.c_void_p), F.shape[0], weight_p, safety_hor, rho, threads)
            return
        self.h = self.L.orc_create(shape.encode(), _p(pp), _p(poly), 0 if poly is None else poly.size // 2, weight_p, safety_hor, rho, threads)
        self.N = 0

    def __del__(self):
        try:
            if self.h:
                self.L.orc_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def set_threads(self, n):
        self.L.orc_set_threads(self.h, int(n))

    def set_points(self, pts):
        pts = _f64(pts)
        self.L.orc_set_points(self.h, _p(pts), pts.shape[0], pts.shape[1])
        self.P = pts.shape[0]

    def set_traj(self, T, coeffs_colmajor):
        T = _f64(T)
        c = _f64(coeffs_colmajor).reshape(-1)
        self.N = T.shape[0]
        self.L.orc_set_traj(self.h, self.N, _p(T), _p(c))

    def duration(self):
        return self.L.orc_traj_duration(self.h)

    def traj_pos(self, t):
        out = np.empty(3)
        self.L.orc_traj_pos(self.h, float(t), _p(out))
        return out

    def traj_vel(self, t):
        out = np.empty(3)
        self.L.orc_traj_vel(self.h, float(t), _p(out))
        return out

    def sdf_at(self, p, t):
        p = _f64(p)
        return self.L.orc_sdf_at(self.h, _p(p), float(t))

    def choice_t_init(self, p, dt=0.15):
        p = _f64(p)
        return self.L.orc_choice_t_init(self.h, _p(p), dt)

    def gradient_descent(self, p, tmin, tmax, x0):
        p = _f64(p)
        fx = C.c_double()
        x = C.c_double()
        self.L.orc_gradient_descent(self.h, _p(p), tmin, tmax, x0, C.cast(C.byref(fx), dp), C.cast(C.byref(x), dp))
        return fx.value, x.value

    def count_evals(self, on=True):
        self.L.orc_count_evals(self.h, 1 if on else 0)

    def eval_count(self):
        return int(self.L.orc_eval_count(self.h))

    def query_outer(self, pts):
        pts = _f64(pts).reshape(-1, 3)
        n = pts.shape[0]
        sdf, ts, g = np.empty(n), np.empty(n), np.empty((n, 3))
        self.L.orc_query_outer(self.h, n, _p(pts), _p(sdf), _p(ts), _p(g))
        return sdf, ts, g

    def query(self, pts):
        pts = _f64(pts).reshape(-1, 3)
        n = pts.shape[0]
        sdf, ts, g = np.empty(n), np.empty(n), np.empty((n, 3))
        rounds = np.zeros(n, dtype=np.int32)
        self.L.orc_query(self.h, n, _p(pts), _p(sdf), _p(ts), _p(g), rounds.ctypes.data_as(C.POINTER(C.c_int)))
        return sdf, ts, g, rounds

    def cost_grad(self, T, coeffs_colmajor, cost0=0.0, gradT0=None, gradC0=None, per_point=False):
        T = _f64(T)
        c = _f64(coeffs_colmajor).reshape(-1)
        N = T.shape[0]
        cost = C.c_double(cost0)
        gT = np.zeros(N) if gradT0 is None else _f64(gradT0).copy()
        gC = np.zeros(18 * N) if gradC0 is None else _f64(gradC0).reshape(-1).copy()
        pp = np.empty((self.P, 7)) if per_point else None
        inside = self.L.orc_cost_grad(self.h, N, _p(T), _p(c), C.cast(C.byref(cost), dp), _p(gT), _p(gC), _p(pp))
        return cost.value, gT, gC, pp, int(inside)

    def time_cost_grad(self, T, coeffs_colmajor, warm=1, reps=3):
        T = _f64(T)
        c = _f64(coeffs_colmajor).reshape(-1)
        cost = C.c_double()
        sec = self.L.orc_time_cost_grad(self.h, T.shape[0], _p(T), _p(c), warm, reps, C.cast(C.byref(cost), dp))
        return sec, cost.value

    def set_conditions(self, init_s, final_s, N):
        i_s = _f64(np.asarray(init_s).T).reshape(-1)
        f_s = _f64(np.asarray(final_s).T).reshape(-1)
        self.N = N
        self.L.orc_set_conditions(self.h, _p(i_s), _p(f_s), N)

    def evaluate(self, x):
        x = _f64(x)
        g = np.empty_like(x)
        f = self.L.orc_evaluate(self.h, _p(x), _p(g), x.shape[0])
        return f, g

    def last_costs(self):
        out = np.empty(3)
        self.L.orc_last_costs(self.h, _p(out))
        return out

    def get_coeffs(self):
        T = np.empty(self.N)
        b = np.empty(18 * self.N)
        self.L.orc_get_coeffs(self.h, _p(T), _p(b))
        return T, b

    def lbfgs(self, x0, mem_size=16, past=3, delta=1e-6, g_epsilon=0.0, max_iterations=0, min_step=1e-32):
        x = _f64(x0).copy()
        stats = np.zeros(4)
        ret = self.L.orc_lbfgs(self.h, _p(x), x.shape[0], mem_size, past, delta, g_epsilon, max_iterations, min_step, _p(stats))
        return ret, x, dict(f=stats[0], iters=int(stats[1]), evals=int(stats[2]), seconds=stats[3])


def sincos(x, variant="default"):
    x = _f64(x).reshape(-1)
    s, c = np.empty_like(x), np.empty_like(x)
    lib(variant).orc_sincos(x.size, _p(x), _p(s), _p(c))
    return s, c


def atan2(y, x, variant="default"):
    y, x = _f64(y).reshape(-1), _f64(x).reshape(-1)
    out = np.empty_like(x)
    lib(variant).orc_atan2(x.size, _p(y), _p(x), _p(out))
    return out


def num_procs():
    return lib().orc_num_procs()
