"""CPU: the pose-sampled obstacle penalty's definition pieces without a GPU — host::pose_penalty (csrc/host/minco.hpp, compiled with g++
as the runtime unit is) against the oracle's restatement (oracle/pose_oracle.py) bit for bit; the oracle's gather box against the
extraction's rule (k3_points); grad_cost_p's filter and smoothed-L1 regimes at their edges; and the cost's gradient in c and T against
central differences."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import k3_points, oracle_py, pose_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dp = C.POINTER(C.c_double)


@pytest.fixture(scope="module")
def chain(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pose") / "pose_chain.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I",
                           os.path.join(ROOT, "implicit_svsdf_planner_b200", "csrc"), os.path.join(ROOT, "tests", "cpp", "pose_chain.cpp"),
                           "-o", so])
    lib = C.CDLL(so)
    lib.pose_chain.restype = C.c_double
    lib.pose_chain.argtypes = [C.c_double, C.c_int, C.c_int, dp, dp, dp, dp, dp, dp]

    def run(weight, R, T, b, rec):
        T, b, rec = (np.ascontiguousarray(a, dtype=np.float64) for a in (T, b, rec))
        N = T.shape[0]
        gC, gT, part = np.zeros(18 * N), np.zeros(N), np.zeros(N)
        p = lambda a: a.ctypes.data_as(dp)  # noqa: E731
        cost = lib.pose_chain(weight, R, N, p(T), p(b), p(rec), p(gC), p(gT), p(part))
        return cost, gT, gC

    return run


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.uint64)


@pytest.mark.parametrize("N", [1, 2, 8, 64])
@pytest.mark.parametrize("R", [1, 4, 64])
def test_chain_rule_is_the_restatement(chain, N, R):
    """Random records, a third of them inactive (costp <= 0, including -0.0 and 0.0): the C++ and the Python sums agree bit for bit."""
    rng = np.random.default_rng(1000 * N + R)
    T = rng.uniform(0.2, 3.0, N)
    b = rng.normal(0, 2, 18 * N)
    rec = rng.normal(0, 1, (N * (R + 1), 4))
    rec[:, 0] = np.abs(rec[:, 0]) * 5
    off = rng.random(N * (R + 1)) < 0.33
    rec[off, 0] = rng.choice([0.0, -0.0, -1.0], off.sum())
    c1, gT1, gC1 = chain(60.0, R, T, b, rec)
    c2, gT2, gC2 = pose_oracle.accumulate(60.0, R, T, b, rec)
    assert np.array_equal(bits([c1]), bits([c2]))
    assert np.array_equal(bits(gT1), bits(gT2)) and np.array_equal(bits(gC1), bits(gC2))
    # an inactive sample adds nothing, not even +0.0: with every record inactive the gradients keep their -0.0 / +0.0 start
    rec[:, 0] = 0.0
    c3, gT3, gC3 = chain(60.0, R, T, b, rec)
    assert c3 == 0.0 and not gT3.any() and not gC3.any()


def small_map(seed=0, X=30, Y=24, Z=5, lo=(-5.0, -12.0, -2.5), p=0.15):
    rng = np.random.default_rng(seed)
    occ = rng.random((X, Y, Z)) < p
    lo = np.array(lo)
    return k3_points.GridMap3D(lo, lo + np.array([X, Y, Z]), 1.0, occ)


def test_box_is_the_extractions_rule():
    """index_box = getGridIndex(projInMap(c -+ half)) of k3_points, for centres inside, on the edges of and outside the map."""
    gm = small_map()
    rng = np.random.default_rng(4)
    for _ in range(2000):
        c = rng.uniform(gm.boundary_min - 8, gm.boundary_max + 8)
        h = rng.uniform(0.1, 12.0, 3)
        box = pose_oracle.index_box(gm, c, h)
        lo_i = gm.grid_index(gm.proj_in_map(c - h))
        hi_i = gm.grid_index(gm.proj_in_map(c + h))
        assert box == [(lo_i[a], hi_i[a]) for a in range(3)]


def test_filter_keeps_equality_and_z_follows_the_yaw():
    """A voxel with |p_rel_a| = half_a is kept, one beyond is skipped; the z range is centred on the yaw (c_z - yaw), so the yaw picks
    one layer, all of them or none."""
    gm = small_map(p=0.0)
    gm.occ[10, 12, :] = True  # centres (5.5, 0.5, -2 .. 2)
    pos = [3.5, 0.5, 0.0]  # yaw 0: p_rel = (2, 0, c_z)
    _, kept, _ = pose_oracle.grad_cost_p(gm, "Circle", pos, (2.0, 1.0, 0.5), 0.7, with_cells=True)
    assert kept == [(10, 12, 2)]  # |p_rel_x| = 2 = half kept; only the layer at z = 0
    _, kept, _ = pose_oracle.grad_cost_p(gm, "Circle", pos, (1.999, 1.0, 0.5), 0.7, with_cells=True)
    assert kept == []
    _, kept, _ = pose_oracle.grad_cost_p(gm, "Circle", pos, (2.0, 1.0, 3.0), 0.7, with_cells=True)
    assert kept == [(10, 12, k) for k in range(5)]
    _, kept, _ = pose_oracle.grad_cost_p(gm, "Circle", [3.5, 0.5, 40.0], (8.5, 8.5, 8.5), 0.7, with_cells=True)
    assert kept == []  # a yaw far from every layer: the box's z range is clipped to the top layer, the filter drops it


def test_smoothed_l1_regimes():
    """safety_hor - sdf below 0, equal to 0, in (0, mu] and above mu: inactive, inactive (f = 0), the cubic, the linear part."""
    gm = small_map(p=0.0)
    gm.occ[10, 12, 2] = True  # centre (5.5, 0.5, 0.5)
    # Circle (radius r): sdf = distance - r; put the robot at distance r + safety_hor - x for x in the four regimes
    radius = -float(oracle_py.shape_sdf("Circle", np.zeros((1, 3)))[0])
    for x, active in ((-0.01, False), (0.0, False), (0.004, True), (0.3, True)):
        d = radius + 0.7 - x
        rec = pose_oracle.grad_cost_p(gm, "Circle", [5.5 - d, 0.5, 0.5], (8.5, 8.5, 8.5), 0.7)
        assert (rec[0] > 0) == active, (x, rec)


def fd_cost(gm, T, co, R, half):
    return pose_oracle.pose_penalty(gm, "star", T, co, 60.0, R, half, 0.7)[0]


def test_gradient_matches_central_differences():
    gm = small_map(seed=2, p=0.08)
    T = np.array([1.3, 0.9])
    b = np.zeros((12, 3))
    b[0] = [2.0, 0.0, 0.1]
    b[1] = [1.5, 0.3, 0.2]
    b[6] = [3.95, 0.6, 0.36]
    b[7] = [1.4, 0.2, 0.1]
    co = np.ascontiguousarray(b.T).reshape(-1)
    R, half = 4, (8.5, 8.5, 8.5)
    cost, gT, gC, rec = pose_oracle.pose_penalty(gm, "star", T, co, 60.0, R, half, 0.7)
    assert cost > 0 and (rec[:, 0] > 0).sum() >= 4
    h = 1e-6
    for e in list(range(0, 18 * 2, 5)):
        cp, cm = co.copy(), co.copy()
        cp[e] += h
        cm[e] -= h
        fd = (fd_cost(gm, T, cp, R, half) - fd_cost(gm, T, cm, R, half)) / (2 * h)
        assert abs(fd - gC[e]) <= 1e-4 * max(1.0, abs(gC[e])), (e, fd, gC[e])
    for i in range(2):
        Tp, Tm = T.copy(), T.copy()
        Tp[i] += h
        Tm[i] -= h
        fd = (fd_cost(gm, Tp, co, R, half) - fd_cost(gm, Tm, co, R, half)) / (2 * h)
        assert abs(fd - gT[i]) <= 1e-4 * max(1.0, abs(gT[i])), (i, fd, gT[i])
