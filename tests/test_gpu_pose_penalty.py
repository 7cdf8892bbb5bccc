"""GPU (-m gpu): the pose-sampled obstacle penalty (svsdf_set_pose_penalty) — off is today's bits and launches; svsdf_pose_penalty_eval's
sample records and its cost and gradient equal the oracle (oracle/pose_oracle.py) bit for bit in the strict build; the callback is the
safety term plus the penalty and matches central differences; svsdf_optimize, svsdf_optimize_lockstep and svsdf_optimize_device agree
bit for bit per problem; refused settings keep the previous one; a box over the whole map has no cap; and between two samples the
penalty does not see an obstacle that the SVSDF term and map_clearance see (the tunnel effect)."""
import os
import sys

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api
from oracle import k3_points, pose_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_gpu_lockstep as L  # noqa: E402
import test_gpu_optimize_device as OD  # noqa: E402  (its problems, comparison and parametrisation)

pytestmark = pytest.mark.gpu

PARAMS = OD.PARAMS
KS = 3  # map kernel size (the penalty reads the occupancy bits only)
SHAPES = [("star", (0.0, 0.0, 0.0)), ("star", (0.4, -0.3, 25.0)), ("sdHorseshoe", (0.0, 0.0, 0.0)), ("Circle", (0.2, 0.1, 10.0)),
          ("Polygon", (0.0, 0.0, 0.0))]


def grid_map(seed=5, X=210, Y=36, Z=4, lo=(-10.0, -16.0, -2.0), res=1.0, probs=None):
    """A multi-layer map over test_gpu_optimize_device's problems: every query point's column occupied in one seeded layer, plus
    seeded clutter."""
    rng = np.random.default_rng(seed)
    occ = np.zeros((X, Y, Z), dtype=bool)
    lo = np.array(lo, dtype=np.float64)
    for p in probs if probs is not None else OD.mixed_problems(big=False):
        for x, y in p["points"][:, :2]:
            i, j = int((x - lo[0]) // res), int((y - lo[1]) // res)
            if 0 <= i < X and 0 <= j < Y:
                occ[i, j, rng.integers(Z)] = True
    occ |= rng.random((X, Y, Z)) < 0.01
    return k3_points.GridMap3D(boundary_min=lo, boundary_max=lo + np.array([X, Y, Z]) * res, res=float(res), occ=occ)


def set_map(ctx, gm):
    X, Y, Z = gm.size
    ctx.set_map3d(k3_points.generate_map_kernel(gm, KS), X, Y, Z, KS, gm.boundary_min, gm.res)


def traj_of(p):
    T = api.forward_T(p["x0"][:p["N"]])
    b, *_ = api.minco_forward(p["init_s"], p["final_s"], p["x0"][p["N"]:].reshape(-1, 3).T, T)
    return T, np.ascontiguousarray(b.T).reshape(-1)


def pose_ctx(shape, pp=(0.0, 0.0, 0.0), strict=True, gm=None, **kw):
    ctx = L.ctx_for(shape, pp, strict)
    set_map(ctx, gm if gm is not None else grid_map())
    ctx.set_pose_penalty(**kw)
    return ctx


@pytest.mark.parametrize("strict", [True, False])
@pytest.mark.parametrize("shape,pp", SHAPES)
def test_eval_equals_the_oracle(shape, pp, strict):
    """svsdf_pose_penalty_eval's records, cost and gradient: the oracle's bits (strict), within rounding (fast)."""
    gm = grid_map()
    ctx = pose_ctx(shape, pp, strict, gm)
    for p, R, half in ((OD.problem(8, 40, 13), 4, (8.5, 8.5, 8.5)), (OD.problem(3, 1, 12), 16, (3.0, 2.0, 0.7))):
        T, co = traj_of(p)
        cost, gT, gC, rec = ctx.pose_penalty(T, co, dict(weight=60.0, integralIntervs=R, half=half), samples=True)
        ro = pose_oracle.records(gm, shape, T, co, R, half, 0.7, pp)
        assert (ro[:, 0] > 0).any()
        c_o, gT_o, gC_o = pose_oracle.accumulate(60.0, R, T, co, ro)
        if strict:
            assert np.array_equal(L.bits(rec), L.bits(ro)), np.argwhere(rec != ro)[:5]
            assert np.array_equal(L.bits([cost]), L.bits([c_o]))
            assert np.array_equal(L.bits(gT), L.bits(gT_o)) and np.array_equal(L.bits(gC), L.bits(gC_o))
        else:
            # contraction moves the functors' central differences (dx = 1e-6) by up to ~1e-8 relative
            np.testing.assert_allclose(rec, ro, rtol=1e-6, atol=1e-7)
            np.testing.assert_allclose(cost, c_o, rtol=1e-7)
            np.testing.assert_allclose(gC, gC_o, rtol=1e-6, atol=1e-6 * np.abs(gC_o).max())
    ctx.close()


def test_off_is_today():
    """Set, then clear: evaluate, optimize, lockstep and device give the bits and the launches of a context that never set it."""
    probs = OD.mixed_problems(big=False)
    gm = grid_map()

    def run(ctx):
        out, launches = [], []
        for p in probs:
            ctx.set_points(p["points"])
            ctx.set_boundary(p["init_s"], p["final_s"], p["N"])
            n0 = ctx.kernel_launches()
            f, g = ctx.evaluate(p["x0"])
            launches.append(ctx.kernel_launches() - n0)
            out.append((f, g, ctx.last_costs()))
        n0 = ctx.kernel_launches()
        single = [L.run_single(ctx, p, PARAMS) for p in probs]
        n1 = ctx.kernel_launches()
        lock = ctx.optimize_lockstep(probs, PARAMS, max_in_flight=3)
        n2 = ctx.kernel_launches()
        dev = ctx.optimize_device(probs, PARAMS)
        n3 = ctx.kernel_launches()
        return out, launches + [n1 - n0, n2 - n1, n3 - n2], single, lock, dev

    fresh = L.ctx_for("star")
    set_map(fresh, gm)
    ref = run(fresh)
    ctx = pose_ctx("star", gm=gm)
    on = [L.run_single(ctx, p, PARAMS) for p in probs]
    assert any(a["final_cost"] != b["final_cost"] for a, b in zip(on, ref[2]))  # the setting did something
    ctx.set_pose_penalty(None)
    got = run(ctx)
    for (f, g, c), (f2, g2, c2) in zip(ref[0], got[0]):
        assert np.array_equal(L.bits(f2), L.bits(f)) and np.array_equal(L.bits(g2), L.bits(g))
        assert np.array_equal(L.bits(c2), L.bits(c))
    assert got[1] == ref[1]
    OD.assert_same(got[2], ref[2], "optimize after clearing")
    OD.assert_same(got[3][0], ref[3][0], "lockstep after clearing")
    OD.assert_same(got[4][0], ref[4][0], "device after clearing")
    ctx.close()
    fresh.close()


@pytest.mark.parametrize("N", [2, 5])
def test_callback_cost_and_gradient(N):
    """Zero query points: the callback is energy + rho sum(T) + the penalty; cost_pos is the penalty; the gradient matches central
    differences in tau and xi.  With dynamics on too, the callback adds both."""
    p = OD.problem(N, 0, 70 + N)
    gm = grid_map(probs=[OD.problem(N, 60, 70 + N)])
    ctx = L.ctx_for("star")
    set_map(ctx, gm)
    ctx.set_points(np.zeros((0, 3)))
    ctx.set_boundary(p["init_s"], p["final_s"], N)
    f_off, _ = ctx.evaluate(p["x0"])
    ctx.set_pose_penalty()
    f_on, g_on = ctx.evaluate(p["x0"])
    T, co = traj_of(p)
    pen = ctx.pose_penalty(T, co)[0]
    assert pen > 0
    assert abs(f_on - (f_off + pen)) <= 1e-12 * abs(f_on)
    costs = ctx.last_costs()
    assert abs(costs[0] - pen) <= 1e-12 * pen and costs[2] == f_on
    x = p["x0"]
    scale = np.abs(g_on).max()
    for e in range(x.shape[0]):
        h = 1e-6 * max(1.0, abs(x[e]))
        xp, xm = x.copy(), x.copy()
        xp[e] += h
        xm[e] -= h
        fd = (ctx.evaluate(xp)[0] - ctx.evaluate(xm)[0]) / (2 * h)
        assert abs(fd - g_on[e]) <= 1e-5 * max(abs(g_on[e]), 1e-2 * scale), (e, fd, g_on[e])
    ctx.set_dynamics(vmax=0.8, omgmax=0.3)
    f_both, _ = ctx.evaluate(p["x0"])
    dyn = api.dynamics_penalty(T, co, dict(vmax=0.8, omgmax=0.3))[0]
    assert dyn > 0 and abs(f_both - (f_on + dyn)) <= 1e-12 * abs(f_both)
    assert abs(ctx.last_costs()[0] - pen) <= 1e-12 * pen  # the dynamics penalty counts in cost_other
    ctx.close()


@pytest.mark.parametrize("strict", [True, False])
@pytest.mark.parametrize("shape,pp", SHAPES)
def test_three_back_ends_agree(shape, pp, strict):
    ctx = pose_ctx(shape, pp, strict)
    probs = OD.mixed_problems(big=(shape == "star" and pp[2] == 0.0))
    for dyn in (None, dict(vmax=0.8, omgmax=0.3)):
        ctx.set_dynamics(dyn)
        ref = [L.run_single(ctx, p, PARAMS) for p in probs]
        lock, r_lock = ctx.optimize_lockstep(probs, PARAMS)
        got, rounds = ctx.optimize_device(probs, PARAMS)
        OD.assert_same(got, ref, (shape, pp, strict, dyn, "single"))
        OD.assert_same(got, lock, (shape, pp, strict, dyn, "lockstep"))
        assert rounds == r_lock == max(r["evaluations"] for r in ref)
    ctx.close()


@pytest.mark.parametrize("strict", [True, False])
def test_back_ends_agree_scaled_and_in_flight(strict):
    """A scale schedule (the penalty stays rigid: its records do not change), max_in_flight 1 and 3, and the batch pool."""
    ctx = pose_ctx("star", strict=strict)
    probs = OD.mixed_problems(big=False)
    T, co = traj_of(probs[2])
    rigid = ctx.pose_penalty(T, co, samples=True)
    ctx.set_scale(**api.EXAMPLE_SCALE)
    scaled = ctx.pose_penalty(T, co, samples=True)
    assert np.array_equal(L.bits(rigid[3]), L.bits(scaled[3])) and rigid[0] == scaled[0]
    ref = [L.run_single(ctx, p, PARAMS) for p in probs]
    OD.assert_same(ctx.optimize_device(probs, PARAMS)[0], ref, ("scaled", strict, "device"))
    ctx.set_scale(None)
    ref = [L.run_single(ctx, p, PARAMS) for p in probs]
    for m in (1, 3):
        OD.assert_same(ctx.optimize_lockstep(probs, PARAMS, max_in_flight=m)[0], ref, ("lockstep", m))
        OD.assert_same(ctx.optimize_device(probs, PARAMS, max_in_flight=m)[0], ref, ("device", m))
    ctx.close()


def test_refusals_keep_the_setting():
    p = OD.problem(8, 40, 13)
    T, co = traj_of(p)
    mesh = L.ctx_for("star_obj_mesh")
    with pytest.raises(api.SvsdfError):
        mesh.set_pose_penalty()
    mesh.close()
    ctx = L.ctx_for("star")
    ctx.set_points(p["points"])
    ctx.set_boundary(p["init_s"], p["final_s"], p["N"])
    ctx.set_pose_penalty()
    n0 = ctx.kernel_launches()
    with pytest.raises(api.SvsdfError):  # no map: refused before any launch
        ctx.evaluate(p["x0"])
    with pytest.raises(api.SvsdfError):
        ctx.optimize_device([p], PARAMS)
    with pytest.raises(api.SvsdfError):
        ctx.optimize_lockstep([p], PARAMS)
    gm = grid_map()
    flat = k3_points.GridMap3D(gm.boundary_min, gm.boundary_max, gm.res, gm.occ[:, :, :1].copy())
    ctx.set_map(k3_points.generate_map_kernel_2d(flat, KS), flat.size[0], flat.size[1], KS, flat.boundary_min[:2], flat.res)
    with pytest.raises(api.SvsdfError):  # a 2-D map
        ctx.evaluate(p["x0"])
    with pytest.raises(api.SvsdfError):
        ctx.pose_penalty(T, co)
    assert ctx.kernel_launches() == n0
    set_map(ctx, gm)
    f, g = ctx.evaluate(p["x0"])
    for bad in (dict(weight=-1.0), dict(integralIntervs=0), dict(integralIntervs=65), dict(half=0.0), dict(half=(1.0, -1.0, 1.0)),
                dict(weight=float("nan")), dict(half=float("inf"))):
        with pytest.raises(api.SvsdfError):
            ctx.set_pose_penalty(**bad)
        assert ctx.pose == api.pose_penalty().as_dict()
        f2, g2 = ctx.evaluate(p["x0"])
        assert np.array_equal(L.bits(f2), L.bits(f)) and np.array_equal(L.bits(g2), L.bits(g))
    ctx.close()


def test_whole_map_box_has_no_cap():
    """A box over the whole map (thousands of occupied cells per sample) equals the oracle."""
    gm = grid_map(seed=9, X=60, Y=40, Z=3, lo=(-10.0, -20.0, -1.5))
    gm.occ |= np.random.default_rng(3).random(gm.occ.shape) < 0.5
    ctx = pose_ctx("star", gm=gm)
    p = OD.problem(3, 0, 12)
    T, co = traj_of(p)
    prm = dict(weight=60.0, integralIntervs=2, half=(500.0, 500.0, 500.0))
    cost, gT, gC, rec = ctx.pose_penalty(T, co, prm, samples=True)
    ro = pose_oracle.records(gm, "star", T, co, 2, prm["half"], 0.7)
    assert np.array_equal(L.bits(rec), L.bits(ro))
    assert gm.occ.sum() > 3000
    ctx.close()


def test_tunnel_effect():
    """A fast straight R = 1 trajectory past one occupied column lying between its two samples: the pose cost is 0, map_clearance lists
    the column as colliding, and the SVSDF cost with that cell as the query point is > 0."""
    X, Y, Z, res = 40, 20, 1, 1.0
    occ = np.zeros((X, Y, Z), dtype=bool)
    occ[20, 10, 0] = True  # centre (10.5, 0.5, 0.5) with lo = (-10, -10, 0)
    lo = np.array([-10.0, -10.0, 0.0])
    gm = k3_points.GridMap3D(lo, lo + np.array([X, Y, Z]) * res, res, occ)
    ctx = L.ctx_for("Circle", (0.0, 0.0, 0.0))
    set_map(ctx, gm)
    b = np.zeros((6, 3))
    b[0] = [-5.0, 0.5, 0.5]
    b[1] = [30.0, 0.0, 0.0]  # x from -5 to 25 in one second: samples at x = -5 and 25, the column at x = 10.5
    T, co = np.array([1.0]), np.ascontiguousarray(b.T).reshape(-1)
    cost, _, _ = ctx.pose_penalty(T, co, dict(integralIntervs=1, half=(8.5, 8.5, 8.5)))
    assert cost == 0.0
    clr = ctx.map_clearance(T, co)
    assert clr.n_colliding == 1 and tuple(clr.ij[0]) == (20, 10)
    ctx.set_points(np.array([[10.5, 0.5, 0.0]]))
    assert ctx.cost_grad(T, co)[0] > 0
    ctx.close()
