"""Seeded synthetic workloads for the SVSDF cost/gradient path (BASELINE.json configs 1-5).

The reference ships only tiny scenes (O(100) query points, SURVEY.md §0); the 2k / 200k / 500k-point
configs are synthetic scale-ups defined here (SURVEY.md §8d).  Inputs taken from the reference's fixtures:
start/goal of ``src/plan_manager/pcds/trajectory_<shape>.txt``, the yaml constants of
``src/plan_manager/config/star.yaml`` (weight_p 60, safety_hor 0.7, rho 3.8, inittime 2.5, kernel_size 17,
occupancy_resolution 1.0), and the way ``plan_manager.cpp:128-175`` builds the query set (occupied cell
centres inside AABBs of half-size kernel_size*res/3 around the waypoints).

numpy only; no oracle, no CUDA.  The spline here is a dense numpy solve of the MINCO_S3NU system
(minco.hpp:433-513) and is used only to lay out the scene (corridor carving) and to provide x0.
"""
from __future__ import annotations

import dataclasses
import math
import os

import numpy as np

# src/plan_manager/pcds/trajectory_<shape>.txt (Start / End, xy)
START_GOAL = {
    "star": ((4.3987178802490234, 4.7499313354492188), (20.23274040222168, 64.403488159179688)),
    "sdHorseshoe": ((21.929414749145508, 61.368782043457031), (3.7336540222167969, 2.9125022888183594)),
}

# src/plan_manager/config/star.yaml
YAML = dict(weight_p=60.0, safety_hor=0.7, rho=3.8, inittime=2.5, kernel_size=17, occupancy_resolution=1.0,
            # the back end's speed and yaw-rate limits (api.yaml_dynamics; off unless a context sets them)
            vmax=10.0, omgmax=10.0, weight_v=10.0, weight_omg=10.0, smoothingEps=1.0e-2, integralIntervs=4)

SEED_TRAJ = 20240501
SEED_MAP = 20240502
SEED_BATCH = 20240503


def _rng(seed: int) -> np.random.Generator:
    return np.random.Generator(np.random.MT19937(seed))


def minco_dense(init_s: np.ndarray, final_s: np.ndarray, q: np.ndarray, T: np.ndarray) -> np.ndarray:
    """MINCO_S3NU coefficients b (6N x 3) by a dense solve of the system of minco.hpp:433-513."""
    N = T.shape[0]
    A = np.zeros((6 * N, 6 * N))
    b = np.zeros((6 * N, 3))
    A[0, 0] = 1.0
    A[1, 1] = 1.0
    A[2, 2] = 2.0
    b[0] = init_s[:, 0]
    b[1] = init_s[:, 1]
    b[2] = init_s[:, 2]
    for i in range(N - 1):
        t1 = T[i]
        t2, t3, t4, t5 = t1**2, t1**3, t1**4, t1**5
        r = 6 * i
        A[r + 3, r + 3 : r + 6] = [6.0, 24.0 * t1, 60.0 * t2]
        A[r + 3, r + 9] = -6.0
        A[r + 4, r + 4 : r + 6] = [24.0, 120.0 * t1]
        A[r + 4, r + 10] = -24.0
        A[r + 5, r : r + 6] = [1.0, t1, t2, t3, t4, t5]
        A[r + 6, r : r + 6] = [1.0, t1, t2, t3, t4, t5]
        A[r + 6, r + 6] = -1.0
        A[r + 7, r + 1 : r + 6] = [1.0, 2 * t1, 3 * t2, 4 * t3, 5 * t4]
        A[r + 7, r + 7] = -1.0
        A[r + 8, r + 2 : r + 6] = [2.0, 6 * t1, 12 * t2, 20 * t3]
        A[r + 8, r + 8] = -2.0
        b[r + 5] = q[:, i]
    t1 = T[N - 1]
    t2, t3, t4, t5 = t1**2, t1**3, t1**4, t1**5
    A[6 * N - 3, 6 * N - 6 :] = [1.0, t1, t2, t3, t4, t5]
    A[6 * N - 2, 6 * N - 5 :] = [1.0, 2 * t1, 3 * t2, 4 * t3, 5 * t4]
    A[6 * N - 1, 6 * N - 4 :] = [2.0, 6 * t1, 12 * t2, 20 * t3]
    b[6 * N - 3] = final_s[:, 0]
    b[6 * N - 2] = final_s[:, 1]
    b[6 * N - 1] = final_s[:, 2]
    return np.linalg.solve(A, b)


def eval_traj_xy(b: np.ndarray, T: np.ndarray, ts: np.ndarray) -> np.ndarray:
    """Positions (x, y, yaw) of the piecewise quintic at global times ts (vectorised, scene layout only)."""
    N = T.shape[0]
    starts = np.concatenate([[0.0], np.cumsum(T)[:-1]])
    idx = np.clip(np.searchsorted(np.cumsum(T), ts, side="left"), 0, N - 1)
    s = ts - starts[idx]
    pw = np.stack([s**k for k in range(6)], axis=1)  # (M, 6)
    c = b.reshape(N, 6, 3)[idx]  # (M, 6, 3)
    return np.einsum("mk,mkd->md", pw, c)


def forward_T(tau: np.ndarray) -> np.ndarray:
    """back_end_optimizer.hpp:213-226."""
    return np.where(tau > 0.0, (0.5 * tau + 1.0) * tau + 1.0, 1.0 / ((0.5 * tau - 1.0) * tau + 1.0))


def backward_T(T: np.ndarray) -> np.ndarray:
    """back_end_optimizer.hpp:228-241."""
    T = np.asarray(T, dtype=np.float64)
    return np.where(T > 1.0, np.sqrt(np.maximum(2.0 * T - 1.0, 0.0)) - 1.0, 1.0 - np.sqrt(np.maximum(2.0 / T - 1.0, 0.0)))


@dataclasses.dataclass
class Scene:
    shape: str
    N: int
    init_s: np.ndarray  # 3x3, column k = k-th derivative of (x, y, yaw) at t=0  (plan_manager.cpp:143-147)
    final_s: np.ndarray
    q: np.ndarray  # 3 x (N-1) interior waypoints
    T: np.ndarray  # N durations
    coeffs: np.ndarray  # MINCO b, 6N x 3 (numpy dense solve; the product/oracle recompute their own)
    points: np.ndarray  # P x 3 (x, y, z); z is zeroed by the cost loop like the reference does
    weight_p: float = YAML["weight_p"]
    safety_hor: float = YAML["safety_hor"]
    rho: float = YAML["rho"]
    poly_params: tuple = (0.0, 0.0, 0.0)
    resolution: float = 0.0

    @property
    def P(self) -> int:
        return int(self.points.shape[0])

    @property
    def x0(self) -> np.ndarray:
        """Decision vector [tau, xi] (back_end_optimizer.cpp:13-19; xi = q flattened column-wise)."""
        return np.concatenate([backward_T(self.T), self.q.T.reshape(-1)])

    def coeffs_colmajor(self) -> np.ndarray:
        """6N x 3 Eigen column-major flat buffer (offset d*6N + 6i + k), as the C-ABI expects."""
        return np.ascontiguousarray(self.coeffs.T).reshape(-1)


def make_trajectory(shape: str = "star", N: int = 8, seed: int = SEED_TRAJ, start=None, goal=None):
    """Boundary states, 7 (N-1) interior waypoints on a seeded perturbed line, yaw in [-pi/2, pi/2], T = 2.5 s."""
    rng = _rng(seed)
    if start is None or goal is None:
        start, goal = START_GOAL.get(shape, START_GOAL["star"])
    start = np.asarray(start, dtype=np.float64)
    goal = np.asarray(goal, dtype=np.float64)
    d = goal - start
    L = float(np.linalg.norm(d))
    n = np.array([-d[1], d[0]]) / max(L, 1e-12)
    q = np.zeros((3, N - 1))
    for i in range(N - 1):
        f = (i + 1) / N
        q[:2, i] = start + f * d + n * rng.uniform(-1.5, 1.5) + (d / max(L, 1e-12)) * rng.uniform(-0.5, 0.5)
        q[2, i] = rng.uniform(-math.pi / 2, math.pi / 2)
    init_s = np.zeros((3, 3))
    final_s = np.zeros((3, 3))
    init_s[:2, 0] = start
    final_s[:2, 0] = goal
    init_s[2, 0] = rng.uniform(-math.pi / 2, math.pi / 2)
    final_s[2, 0] = rng.uniform(-math.pi / 2, math.pi / 2)
    # keep the nominal speed near the reference's scenes (~60 m in N*2.5 s would be too fast for N=8 only if
    # the path were longer): durations are inittime per piece as plan_manager.cpp:186 does.
    T = np.full(N, YAML["inittime"])
    return init_s, final_s, q, T


def make_scene(
    shape: str = "star",
    N: int = 8,
    P: int = 2000,
    seed_traj: int = SEED_TRAJ,
    seed_map: int = SEED_MAP,
    clearance: float = 2.75,
    start=None,
    goal=None,
) -> Scene:
    """Config 1/2/3 style scene: exactly P query points = cell centres of a seeded random occupancy grid inside
    the union of waypoint AABBs (half-size kernel_size*res/3 = 5.67 m), with a corridor of half-width
    ``clearance`` carved around the nominal spline so that most points are outside the swept volume, a few
    percent are within safety_hor of it and a handful are inside (all three branches of the reference's
    getTrueSDFofSweptVolume / smoothedL1 are exercised)."""
    init_s, final_s, q, T = make_trajectory(shape, N, seed_traj, start, goal)
    b = minco_dense(init_s, final_s, q, T)
    half = YAML["kernel_size"] * YAML["occupancy_resolution"] / 3.0
    wps = np.concatenate([init_s[:2, :1], q[:2], final_s[:2, :1]], axis=1).T  # include the end points
    lo = wps.min(axis=0) - half
    hi = wps.max(axis=0) + half
    # dense samples of the nominal path for corridor carving
    D = float(T.sum())
    ts = np.linspace(0.0, D, 4001)
    path = eval_traj_xy(b, T, ts)[:, :2]

    rng = _rng(seed_map)
    # choose the resolution so that the candidate set (in boxes, outside the corridor) is ~3.3x P: count candidates
    # on a coarse 0.25 m grid, then scale (cells ~ 1 / res^2)
    def grid(res):
        nx = int(math.ceil((hi[0] - lo[0]) / res))
        ny = int(math.ceil((hi[1] - lo[1]) / res))
        xs = lo[0] + (np.arange(nx) + 0.5) * res
        ys = lo[1] + (np.arange(ny) + 0.5) * res
        return _candidates(xs, ys, wps, half, path, clearance)

    res = 0.25
    cand = grid(res)
    if cand.shape[0] < 3.0 * P:
        res = 0.25 * math.sqrt(cand.shape[0] / (3.3 * P))
        cand = grid(res)
    if cand.shape[0] < P:
        raise ValueError(f"scene too small for P={P} (candidates={cand.shape[0]})")
    sel = np.sort(rng.choice(cand.shape[0], size=P, replace=False))  # keep grid (row-major) order
    pts = np.zeros((P, 3))
    pts[:, :2] = cand[sel]
    pts[:, 2] = rng.integers(0, 3, size=P) * YAML["occupancy_resolution"]  # stacked voxels; z is ignored by the cost
    return Scene(shape=shape, N=N, init_s=init_s, final_s=final_s, q=q, T=T, coeffs=b, points=pts, resolution=res)


def _candidates(xs, ys, wps, half, path, clearance):
    from scipy.spatial import cKDTree

    gx, gy = np.meshgrid(xs, ys, indexing="xy")  # row-major: y rows, x fastest
    pts = np.stack([gx.ravel(), gy.ravel()], axis=1)
    inbox = np.zeros(pts.shape[0], dtype=bool)
    for w in wps:
        inbox |= (np.abs(pts[:, 0] - w[0]) <= half) & (np.abs(pts[:, 1] - w[1]) <= half)
    pts = pts[inbox]
    d, _ = cKDTree(path).query(pts, k=1)  # distance to the densely sampled nominal path
    return pts[d > clearance]


COORDS_TXT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "coords.txt")


def make_batch_problems(n_problems: int, seed: int = SEED_BATCH, extent=(2.0, 58.0), coords_path: str = COORDS_TXT):
    """BASELINE config 5 start/goal pairs (SURVEY.md §8d): the first min(n, 1000) come from the reference's own
    `src/coords.txt` (1000 rows of 6 uniform[0, 60] numbers; columns 0-1 = start xy, 3-4 = goal xy; a copy travels as
    tests/golden/coords.txt), clipped into `extent`; the rest are uniform in `extent` from mt19937_64(seed).  Pairs shorter
    than 25 m are stretched to 25 m along their own direction (an 8-piece, 20 s trajectory over a few metres is degenerate).
    Returns [n, 4] = (start x, start y, goal x, goal y)."""
    rng = _rng(seed)
    lo, hi = extent
    sg = rng.uniform(lo, hi, size=(n_problems, 4))
    if coords_path and os.path.exists(coords_path) and n_problems > 0:
        c = np.loadtxt(coords_path, delimiter=",")
        m = min(n_problems, c.shape[0])
        sg[:m, 0:2] = c[:m, 0:2]
        sg[:m, 2:4] = c[:m, 3:5]
        sg[:m] = np.clip(sg[:m], lo, hi)
    d = sg[:, 2:] - sg[:, :2]
    L = np.linalg.norm(d, axis=1)
    short = L < 25.0
    u = np.where(L[:, None] > 1e-9, d / np.maximum(L[:, None], 1e-9), np.array([[1.0, 0.0]]))
    sg[short, 2:] = sg[short, :2] + u[short] * 25.0
    # a stretched goal may leave the map: reflect it back along the same direction
    out = ((sg[:, 2:] < lo) | (sg[:, 2:] > hi)).any(axis=1)
    sg[out, 2:] = sg[out, :2] - u[out] * 25.0
    sg[:, 2:] = np.clip(sg[:, 2:], lo, hi)
    return sg


# ---------------------------------------------------------------------------------------------------------------------
# Triangle meshes for the mesh-SDF functor (BasicShape::getonlySDF_igl, Shape.hpp:332-340)
# ---------------------------------------------------------------------------------------------------------------------
def load_obj(path: str):
    """Minimal Wavefront .obj reader (what igl::read_triangle_mesh does for the reference's shapes/*.obj, Shape.hpp:285):
    `v x y z` and `f i[/..] j[/..] k[/..] ...` records, 1-based or negative indices, polygons fan-triangulated.
    Returns (V [nv, 3] float64, F [nf, 3] int32)."""
    V, F = [], []
    with open(path, "r") as fh:
        for line in fh:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "v":
                V.append([float(tok[1]), float(tok[2]), float(tok[3])])
            elif tok[0] == "f":
                idx = []
                for t in tok[1:]:
                    i = int(t.split("/")[0])
                    idx.append(i - 1 if i > 0 else len(V) + i)
                for k in range(1, len(idx) - 1):
                    F.append([idx[0], idx[k], idx[k + 1]])
    return np.asarray(V, dtype=np.float64).reshape(-1, 3), np.asarray(F, dtype=np.int32).reshape(-1, 3)


def extrude_outline(outline_xy: np.ndarray, half_height: float = 0.49, center=(0.0, 0.0)):
    """Closed, outward-oriented slab mesh of a 2-D outline that is star-shaped about `center` (counter-clockwise
    vertices): side quads split into two triangles, caps fanned from the centre — the same kind of thin extrusion the
    reference's shapes/*.obj are (SURVEY.md A.9), generated here so that GPU tests need no reference file.
    Returns (V, F)."""
    o = np.asarray(outline_xy, dtype=np.float64).reshape(-1, 2)
    n = o.shape[0]
    h = float(half_height)
    V = np.zeros((2 * n + 2, 3))
    V[:n, :2] = o
    V[:n, 2] = -h
    V[n : 2 * n, :2] = o
    V[n : 2 * n, 2] = h
    V[2 * n] = [center[0], center[1], -h]
    V[2 * n + 1] = [center[0], center[1], h]
    F = []
    for i in range(n):
        j = (i + 1) % n
        F.append([i, j, n + j])          # side, outward for a CCW outline
        F.append([i, n + j, n + i])
        F.append([2 * n, j, i])          # bottom cap (normal -z)
        F.append([2 * n + 1, n + i, n + j])  # top cap (normal +z)
    return V, np.asarray(F, dtype=np.int32)


def star_outline(r_out: float = 2.8, r_in: float = 1.4, tips: int = 5, n_per_edge: int = 1) -> np.ndarray:
    """Counter-clockwise outline of a `tips`-pointed star (first tip on +y), optionally with extra vertices per edge: a
    synthetic robot outline for the mesh-SDF functor (roughly the reference's star, outer radius 2.8; not its level set)."""
    pts = []
    for k in range(2 * tips):
        ang = np.pi / 2 + k * np.pi / tips
        rad = r_out if k % 2 == 0 else r_in
        pts.append([rad * np.cos(ang), rad * np.sin(ang)])
    pts = np.asarray(pts)
    if n_per_edge > 1:
        out = []
        for i in range(2 * tips):
            a, b = pts[i], pts[(i + 1) % (2 * tips)]
            for q in range(n_per_edge):
                out.append(a + (b - a) * (q / n_per_edge))
        pts = np.asarray(out)
    return pts
