"""GPU (-m gpu): the back end's speed and yaw-rate penalty (svsdf_set_dynamics) — off is today's bits; on, svsdf_evaluate's cost is the
safety callback plus svsdf_dynamics_penalty and its gradient matches central differences; svsdf_optimize, svsdf_optimize_lockstep and
svsdf_optimize_device agree bit for bit per problem; plan_batch is generate_traj per problem; and the penalty lowers the planner's
sampled speed excess on the reference's star scene."""
import os
import sys

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, plan, scenes

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_gpu_lockstep as L  # noqa: E402
import test_gpu_optimize_device as OD  # noqa: E402  (its problems, comparison and parametrisation)

pytestmark = pytest.mark.gpu

# limits the seeded trajectories of test_gpu_lockstep exceed, so that the penalty is active from the start
DYN = dict(vmax=0.8, omgmax=0.3, weight_v=10.0, weight_omg=10.0, smoothingEps=1e-2, integralIntervs=4)
PARAMS = OD.PARAMS


def start_penalty(p, dyn=DYN):
    T = api.forward_T(p["x0"][:p["N"]])
    b, *_ = api.minco_forward(p["init_s"], p["final_s"], p["x0"][p["N"]:].reshape(-1, 3).T, T)
    return api.dynamics_penalty(T, b.T.reshape(-1), dyn)[0]


def test_off_is_today():
    """Set, then clear: svsdf_evaluate, svsdf_optimize and svsdf_optimize_device give the bits of a context that never set dynamics."""
    probs = OD.mixed_problems(big=False)
    fresh = L.ctx_for("star")
    ref_eval = []
    for p in probs:
        fresh.set_points(p["points"])
        fresh.set_boundary(p["init_s"], p["final_s"], p["N"])
        ref_eval.append(fresh.evaluate(p["x0"]) + (fresh.last_costs(),))
    ref_single = [L.run_single(fresh, p, PARAMS) for p in probs]
    ref_dev, _ = fresh.optimize_device(probs, PARAMS)
    ctx = L.ctx_for("star")
    ctx.set_dynamics(**DYN)
    on = [L.run_single(ctx, p, PARAMS) for p in probs]
    assert any(a["final_cost"] != b["final_cost"] for a, b in zip(on, ref_single))  # the setting did something
    ctx.set_dynamics(None)
    for p, (f, g, costs) in zip(probs, ref_eval):
        ctx.set_points(p["points"])
        ctx.set_boundary(p["init_s"], p["final_s"], p["N"])
        f2, g2 = ctx.evaluate(p["x0"])
        assert np.array_equal(L.bits(f2), L.bits(f)) and np.array_equal(L.bits(g2), L.bits(g))
        assert np.array_equal(L.bits(ctx.last_costs()), L.bits(costs))
    OD.assert_same([L.run_single(ctx, p, PARAMS) for p in probs], ref_single, "optimize after clearing")
    OD.assert_same(ctx.optimize_device(probs, PARAMS)[0], ref_dev, "optimize_device after clearing")
    ctx.close()
    fresh.close()


def test_refused_limits_keep_the_setting():
    ctx = L.ctx_for("star")
    p = OD.problem(8, 40, 13)
    ctx.set_dynamics(**DYN)
    ctx.set_points(p["points"])
    ctx.set_boundary(p["init_s"], p["final_s"], p["N"])
    f, g = ctx.evaluate(p["x0"])
    for bad in (dict(vmax=0.0), dict(omgmax=-1.0), dict(weight_v=-1.0), dict(smoothingEps=0.0), dict(integralIntervs=65),
                dict(vmax=float("nan"))):
        with pytest.raises(api.SvsdfError):
            ctx.set_dynamics(**dict(DYN, **bad))
        assert ctx.dynamics == api.dynamics(DYN).as_dict()
        f2, g2 = ctx.evaluate(p["x0"])
        assert np.array_equal(L.bits(f2), L.bits(f)) and np.array_equal(L.bits(g2), L.bits(g))
    ctx.close()


@pytest.mark.parametrize("N", [2, 5])
def test_callback_cost_and_gradient(N):
    """Zero query points: the callback is MINCO's energy + rho sum(T) + the penalty, smooth where no sample's violation is near 0 or mu.
    Its cost is the callback without dynamics plus svsdf_dynamics_penalty; its gradient matches central differences in tau and xi."""
    p = OD.problem(N, 0, 70 + N)
    ctx = L.ctx_for("star")
    ctx.set_points(np.zeros((0, 3)))
    ctx.set_boundary(p["init_s"], p["final_s"], N)
    f_off, _ = ctx.evaluate(p["x0"])
    dyn = dict(DYN, smoothingEps=1e-6)
    ctx.set_dynamics(**dyn)
    f_on, g_on = ctx.evaluate(p["x0"])
    pen = start_penalty(p, dyn)
    assert pen > 0
    assert abs(f_on - (f_off + pen)) <= 1e-12 * abs(f_on)
    costs = ctx.last_costs()
    assert costs[0] == 0.0 and costs[2] == f_on  # no query points: no safety term; the penalty counts in cost_other
    x = p["x0"]
    scale = np.abs(g_on).max()
    for e in range(x.shape[0]):
        h = 1e-6 * max(1.0, abs(x[e]))
        xp, xm = x.copy(), x.copy()
        xp[e] += h
        xm[e] -= h
        fd = (ctx.evaluate(xp)[0] - ctx.evaluate(xm)[0]) / (2 * h)
        assert abs(fd - g_on[e]) <= 1e-6 * max(abs(g_on[e]), 1e-2 * scale), (e, fd, g_on[e])
    ctx.close()


@pytest.mark.parametrize("strict", [True, False])
@pytest.mark.parametrize("shape,pp", [("star", (0.0, 0.0, 0.0)), ("star", (0.4, -0.3, 25.0)), ("sdHorseshoe", (0.0, 0.0, 0.0)),
                                      ("Circle", (0.2, 0.1, 10.0)), ("Polygon", (0.0, 0.0, 0.0))])
def test_three_back_ends_agree(shape, pp, strict):
    ctx = L.ctx_for(shape, pp, strict)
    ctx.set_dynamics(**DYN)
    probs = OD.mixed_problems(big=(shape == "star" and pp[2] == 0.0))
    assert all(start_penalty(p) > 0 for p in probs)
    ref = [L.run_single(ctx, p, PARAMS) for p in probs]
    lock, r_lock = ctx.optimize_lockstep(probs, PARAMS)
    got, rounds = ctx.optimize_device(probs, PARAMS)
    OD.assert_same(got, ref, (shape, pp, strict, "single"))
    OD.assert_same(got, lock, (shape, pp, strict, "lockstep"))
    assert rounds == r_lock == max(r["evaluations"] for r in ref)
    ctx.close()


def test_mesh_scale_and_max_in_flight():
    ctx = L.ctx_for("star_obj_mesh")
    ctx.set_dynamics(**DYN)
    probs = [OD.problem(3, 30, 21), OD.problem(5, 50, 22)]
    prm = api.default_lbfgs_params(max_iterations=6)
    OD.assert_same(ctx.optimize_device(probs, prm)[0], [L.run_single(ctx, p, prm) for p in probs], "mesh")
    OD.assert_same(ctx.optimize_lockstep(probs, prm)[0], [L.run_single(ctx, p, prm) for p in probs], "mesh lockstep")
    ctx.close()
    for strict in (True, False):
        ctx = L.ctx_for("star", strict=strict)
        ctx.set_scale(**api.EXAMPLE_SCALE)
        ctx.set_dynamics(**DYN)
        probs = OD.mixed_problems(big=False)
        ref = [L.run_single(ctx, p, PARAMS) for p in probs]
        OD.assert_same(ctx.optimize_device(probs, PARAMS)[0], ref, ("scaled", strict))
        OD.assert_same(ctx.optimize_lockstep(probs, PARAMS)[0], ref, ("scaled lockstep", strict))
        ctx.close()
    ctx = L.ctx_for("star")
    ctx.set_dynamics(**DYN)
    probs = OD.mixed_problems(big=False)
    ref = [L.run_single(ctx, p, PARAMS) for p in probs]
    for m in (1, 3, 0):
        got, rounds = ctx.optimize_device(probs, PARAMS, max_in_flight=m)
        OD.assert_same(got, ref, ("max_in_flight", m))
    ctx.close()


def test_optimize_batch_pool_carries_each_contexts_setting():
    probs = [OD.problem(8, 40, 81), OD.problem(8, 60, 82), OD.problem(8, 0, 83)]
    on, off = L.ctx_for("star"), L.ctx_for("star")
    on.set_dynamics(**DYN)
    ref_on = [L.run_single(on, p, PARAMS) for p in probs]
    ref_off = [L.run_single(off, p, PARAMS) for p in probs]
    assert any(a["final_cost"] != b["final_cost"] for a, b in zip(ref_on, ref_off))
    for ctx, ref in ((on, ref_on), (off, ref_off)):
        _, X, _, status, _ = api.optimize_batch([ctx], [dict(init_s=p["init_s"], final_s=p["final_s"], x0=p["x0"], points=p["points"])
                                                        for p in probs], 8, PARAMS)
        for k, r in enumerate(ref):
            assert np.array_equal(L.bits(X[k]), L.bits(r["x"])) and status[k] == r["status"], k
    on.close()
    off.close()


# ---- planner ------------------------------------------------------------------------------------------------------------------------
def star_scene():
    g = np.load(os.path.join(HERE, "golden", "map_star_pcd.npz"))
    res, ks = float(g["occupancy_resolution"]), int(g["kernel_size"])
    cmap = plan.gridmap3d_from_cloud(g["points"], res, int(g["sta_threshold"]))
    return g, cmap, dict(kernel_size=ks, traj_parlength=float(g["traj_parlength"]))


def ctx_new(dyn=None):
    ctx = api.Context("star", weight_p=scenes.YAML["weight_p"], safety_hor=scenes.YAML["safety_hor"], rho=scenes.YAML["rho"])
    if dyn is not None:
        ctx.set_dynamics(dyn)
    return ctx


def free_pairs(cmap, n, seed):
    free = np.argwhere(~cmap.occ.any(axis=2))
    rng = np.random.default_rng(seed)
    pick = free[rng.integers(0, len(free), size=(n, 2))]
    xy = cmap.boundary_min[:2] + (pick + 0.5) * cmap.res
    return xy[:, 0].copy(), xy[:, 1].copy()


@pytest.mark.parametrize("n", [12, 256])
def test_plan_batch_is_generate_traj_with_dynamics(n):
    """n < 256 runs the host lock-step back end, n >= 256 the device back end; each problem equals generate_traj's bits, with the same
    `dynamics` report."""
    g, cmap, kw = star_scene()
    st, go = free_pairs(cmap, n, 5 + n)
    st[0], go[0] = g["start"][:2], g["end"][:2]
    dyn = dict(api.yaml_dynamics(scenes.YAML).as_dict(), vmax=1.0, omgmax=1.0)
    ctx = ctx_new(dyn)
    got = plan.plan_batch(ctx, cmap, st, go, **kw)
    checked = 0
    for q in range(n) if n < 256 else list(range(0, n, 37)) + [n - 1]:
        r = plan.generate_traj(ctx_new(dyn), cmap, st[q], go[q], **kw)
        b = got[q]
        assert b["ok"] == r["ok"], q
        if "T" not in r:
            continue
        for key in ("x", "T", "coeffs"):
            assert np.array_equal(L.bits(b[key]), L.bits(r[key])), (q, key)
        assert (b["iterations"], b["evaluations"], b["status"]) == (r["iterations"], r["evaluations"], r["status"]), q
        assert b["dynamics"] == r["dynamics"], q
        checked += 1
    assert checked >= 3
    # without dynamics there is no report
    r = plan.generate_traj(ctx_new(), cmap, g["start"][:2], g["end"][:2], **kw)
    assert "dynamics" not in r
    ctx.close()


def excess(T, coeffs, vmax):
    """sampled integral of max(0, |v| - vmax) dt (trapezoid on plan.sampled_rates' lattice)"""
    s, v, _ = plan.sampled_rates(T, coeffs)
    return float(sum(np.trapezoid(np.maximum(v[i] - vmax, 0.0), s[i]) for i in range(len(T))))


def test_penalty_lowers_the_speed_excess_on_the_star_scene():
    g, cmap, kw = star_scene()
    free = plan.generate_traj(ctx_new(), cmap, g["start"][:2], g["end"][:2], certify=True, **kw)
    assert free["ok"]
    _, v, w = plan.sampled_rates(free["T"], free["coeffs"])
    vmax, omgmax = 0.5 * float(v.max()), 0.5 * float(np.abs(w).max())
    dyn = dict(api.yaml_dynamics(scenes.YAML).as_dict(), vmax=vmax, omgmax=omgmax)
    lim = plan.generate_traj(ctx_new(dyn), cmap, g["start"][:2], g["end"][:2], certify=True, **kw)
    assert lim["ok"]
    e0, e1 = excess(free["T"], free["coeffs"], vmax), excess(lim["T"], lim["coeffs"], vmax)
    print(f"\nstar scene: unconstrained v_peak {v.max():.4f} omg_peak {np.abs(w).max():.4f} cost {free['final_cost']:.6g} "
          f"duration {free['T'].sum():.4f} s clearance {free['clearance']['min_sdf']:.4f}; limits vmax {vmax:.4f} omgmax {omgmax:.4f}: "
          f"v_peak {lim['dynamics']['v_peak']:.4f} omg_peak {lim['dynamics']['omg_peak']:.4f} cost {lim['final_cost']:.6g} "
          f"duration {lim['T'].sum():.4f} s clearance {lim['clearance']['min_sdf']:.4f} collision_free {lim['clearance']['collision_free']}; "
          f"excess integral {e0:.6g} -> {e1:.6g} m")
    assert e1 < e0
