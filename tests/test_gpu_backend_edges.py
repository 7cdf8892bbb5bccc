"""GPU (-m gpu): svsdf_optimize_device at the limits of its inputs.

- Against the mathematics: with g_epsilon = 1e30 every problem takes one evaluation, so the coefficients the device's finish computed
  and the device's cost_at_start (energy + dynamics penalty + rho sum T, no query points) are compared with the 60-digit references of
  test_backend_exact.py, all cases of that file the problems of one call; and svsdf_evaluate's tau gradient (backwardGradT) against
  the 60-digit adjoint times dT/dtau.
- Bit for bit with svsdf_optimize and svsdf_optimize_lockstep, dynamics and the pose penalty on: the warp's lane wrap (N = 31, 32, 33,
  63, 64), a 1 ms piece among 2 s pieces, a start whose duration D is the layer-1 lattice point t (t += 0.15 from 0) just below 300 s
  and one ulp below it, integralIntervs 1 and 64, and 1 200 problems of mixed N through max_in_flight 1, 7, 64, the default (1 024)
  and all at once; strict and FMA builds."""
import os
import sys

import mpmath as mp
import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_backend_exact as X  # noqa: E402  (the 60-digit references and their cases)
import test_gpu_lockstep as L  # noqa: E402
import test_gpu_optimize_device as OD  # noqa: E402
import test_gpu_pose_penalty as PP  # noqa: E402

pytestmark = pytest.mark.gpu

RHO = 3.8
STOP = api.default_lbfgs_params(g_epsilon=1e30)
# observed maxima of error / (u M) on an H100, cost_at_start: 0.0039 (typical_N64); CONTRAST cases 3.3 (loguniform_N64)
C_COST, C_COST_CONTRAST = 0.02, 16.0


def exact_problem(name):
    init_s, final_s, q, T = X.case(name)
    N = len(T)
    x0 = np.r_[api.backward_T(T), q.T.reshape(-1)]
    Tf = api.forward_T(x0[:N])  # the durations the back end works with (forward_T is pinned by test_backend_exact)
    return dict(N=N, init_s=init_s, final_s=final_s, x0=x0, points=np.zeros((0, 3))), q, Tf


def test_device_first_evaluation_is_the_exact_mathematics():
    """All cases of test_backend_exact as the problems of one optimize_device call (N 2 to 64 mixed), under one set of speed limits
    (the median sampled speed and yaw rate over all cases): per problem, the coefficients per piece within C_COEF u Skeel's measure
    (C_CONTRAST on the CONTRAST cases), cost_at_start within C_COST u (|terms| + the coefficients' measure carried through
    |dcost / dc|)."""
    items = [exact_problem(name) for name, _, _ in X.CASES]
    v, w = np.median([X._speeds(Tf, np.ascontiguousarray(api.minco_forward(p["init_s"], p["final_s"], q, Tf)[0].T).reshape(-1), 4)
                      for p, q, Tf in items], axis=0)
    dyn = X._dyn(vmax=float(v), omgmax=float(w), smoothingEps=0.3 * float(v) ** 2, integralIntervs=4)
    ctx = L.ctx_for("star")
    ctx.set_dynamics(dyn)
    got, rounds = ctx.optimize_device([it[0] for it in items], STOP)
    ctx.close()
    assert rounds == 1 and all(g["evaluations"] == 1 for g in got)
    active = 0
    for (name, N, _), (p, q, Tf), g in zip(X.CASES, items, got):
        assert np.array_equal(L.bits(g["T"]), L.bits(Tf))
        mc = X.Minco(p["init_s"], p["final_s"], q, Tf)
        A, Ainv_abs = X.dense(mc)
        Sc = X.coeff_measure(mc, Ainv_abs, A)
        bdev = g["coeffs"].reshape(3, 6 * N).T
        err = X._err(bdev, [v for r in mc.c for v in r]).reshape(6 * N, 3)
        r_coef = X._ratio(X.piece_norms(err, N), X.piece_norms(Sc, N))
        assert r_coef <= (X.C_CONTRAST if name in X.CONTRAST else X.C_COEF), (name, r_coef)
        # the cost of the exact spline at 60 digits
        E, gE, _ = X.energy_exact(mc.c, Tf)
        flat = [mc.c[r][d] for d in range(3) for r in range(6 * N)]  # 18N column-major
        with mp.workdps(X.DPS):
            bx = np.array([float(v) for v in flat])
            dyn_c = sum(X.dyn_piece_cost(dyn, mp.mpf(float(Tf[i])), [[flat[dd * 6 * N + 6 * i + k] for k in range(6)] for dd in range(3)])
                        for i in range(N))
            xcost = E + dyn_c + mp.mpf(RHO) * sum(mp.mpf(float(t)) for t in Tf)
        active += dyn_c > 0
        Ea, _, _ = X.energy_exact(mc.c, Tf, absolute=True)
        m_dyn, _, m_g = X.dyn_measures(dyn, Tf, bx)
        gEa = np.abs(np.array([[float(v) for v in r] for r in gE]))
        meas = float(Ea) + m_dyn + RHO * Tf.sum() + (gEa * Sc).sum() + (m_g.reshape(3, 6 * N).T * Sc).sum()
        r_cost = abs(float(mp.mpf(g["cost_at_start"]) - xcost)) / (X.U * meas)
        print(f"{name}: coef {r_coef:.3g} cost {r_cost:.3g}")
        assert r_cost <= (C_COST_CONTRAST if name in X.CONTRAST else C_COST), (name, r_cost)
    assert active >= len(X.CASES) // 2  # the penalty is on in most problems


def dT_dtau(tau):
    """the tau map's derivative at 60 digits"""
    t = mp.mpf(float(tau))
    return t + 1 if tau > 0 else (1 - t) / (t * t / 2 - t + 1) ** 2


# observed maxima of error / (u M) per piece on an H100: 0.0076 (D299.9_N64); CONTRAST cases 135 (250s_N4, the coefficients' growth
# carried into the adjoint)
C_TAU, C_TAU_CONTRAST = 0.05, 1024.0


def test_evaluate_tau_gradient_is_the_exact_chain():
    """svsdf_evaluate's gradient with no query points and no penalties, d(E + rho sum T) / d tau, against the 60-digit chain: the exact
    adjoint with W = dE/dc and wT = dE/dT + rho, times dT/dtau (backwardGradT).  Per piece within C_TAU u M: M the adjoint's measure
    with the partials' own rounding carried in (H Skeel(c) for dE/dc, 2 |jerk(c)| |jerk(Skeel(c))| + |jerk(Skeel(c))|^2 for dE/dT),
    times |dT/dtau|, plus |the exact gradient|."""
    ctx = L.ctx_for("star")
    ctx.set_points(np.zeros((0, 3)))
    branches = set()
    for name, N, _ in X.CASES:
        p, q, Tf = exact_problem(name)
        branches |= set(p["x0"][:N] > 0)
        ctx.set_boundary(p["init_s"], p["final_s"], N)
        _, g = ctx.evaluate(p["x0"])
        mc = X.Minco(p["init_s"], p["final_s"], q, Tf)
        A, Ainv_abs = X.dense(mc)
        Sc = X.coeff_measure(mc, Ainv_abs, A)
        _, gE, gTE = X.energy_exact(mc.c, Tf)
        with mp.workdps(X.DPS):
            wT = [t + mp.mpf(RHO) for t in gTE]
            _, xT, lam = mc.adjoint(gE, wT)
            dtd = [dT_dtau(t) for t in p["x0"][:N]]
            xg = [a * b for a, b in zip(xT, dtd)]
        ca = np.abs(mc.coeffs())
        _, HS, _ = X.energy_exact(Sc, Tf, absolute=True)
        _, _, tCS = X.energy_exact(ca + Sc, Tf, absolute=True)
        _, _, tC = X.energy_exact(ca, Tf, absolute=True)
        mc._W = np.abs(np.array([[float(v) for v in r] for r in gE])) + np.array([[float(v) for v in r] for r in HS])
        mc._wT = np.abs(np.array([float(v) for v in wT])) + np.array([float(a - b) for a, b in zip(tCS, tC)])
        _, mt = X.adjoint_measures(mc, A, Ainv_abs, lam)
        adt = np.abs(np.array([float(v) for v in dtd]))
        meas = mt * adt + np.abs(np.array([float(v) for v in xg]))
        r = X._ratio(np.abs(X._err(g[:N], xg)), meas)
        print(f"{name}: tau gradient {r:.3g}")
        assert r <= (C_TAU_CONTRAST if name in X.CONTRAST else C_TAU), (name, r)
    assert branches == {True, False}  # both branches of the tau map
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------------------
# bit for bit with the host back ends


def with_durations(N, T, P, seed):
    """test_gpu_optimize_device's problem of N pieces with the durations T (its path) and P points near the result"""
    p = OD.problem(N, 0, seed)
    p["x0"] = np.r_[api.backward_T(np.asarray(T, dtype=np.float64)), p["x0"][N:]]
    Tf, co = PP.traj_of(p)
    p["points"] = L.points_near(Tf, co, P, seed + 1000, spread=2.5) if P else np.zeros((0, 3))
    return p


def lattice_point_below(D=300.0):
    """the last t of `for (t = 0; t <= D; t += 0.15)` below D"""
    t, last = 0.0, 0.0
    while t < D:
        last = t
        t += 0.15
    return last


def durations_summing_to(N, D):
    """N durations near D / N whose sum in order (as the back end accumulates forward_T(tau)) is exactly D; returns the taus"""
    tau = np.full(N, api.backward_T(np.array([D / N]))[0])
    T = api.forward_T(tau)
    s = 0.0
    for t in T[:-1]:
        s += t
    base = api.backward_T(np.array([D - s]))[0]
    for k in range(4096):
        for cand in (base + k * np.spacing(base), base - k * np.spacing(base)):
            if s + api.forward_T(np.array([cand]))[0] == D:
                tau[-1] = cand
                return tau
    raise AssertionError(("no tau gives D", D))


def lattice_problems():
    tk = lattice_point_below()
    out = []
    for D in (tk, np.nextafter(tk, 0.0)):
        tau = durations_summing_to(64, D)
        p = with_durations(64, api.forward_T(tau), 40, 91)
        p["x0"][:64] = tau
        Tf = api.forward_T(tau)
        s = 0.0
        for t in Tf:
            s += t
        assert s == D
        out.append(p)
    return out


EDGE_SETS = {
    "lane_wrap": lambda: [OD.problem(N, 20, 60 + N, dur=2.0) for N in (31, 32, 33, 63, 64)],
    "1ms_piece": lambda: [with_durations(8, np.r_[np.full(4, 2.0), 1e-3, np.full(3, 2.0)], 30, 81),
                          with_durations(33, np.r_[1e-3, np.full(32, 2.0)], 30, 82)],
    "lattice_D": lattice_problems,
}


def edge_ctx(strict, problems, res=4):
    ctx = PP.pose_ctx("star", strict=strict, gm=PP.grid_map(probs=problems), integralIntervs=res)
    ctx.set_dynamics(vmax=0.8, omgmax=0.3, integralIntervs=res)
    return ctx


def three_back_ends(ctx, probs, prm, what):
    ref = [L.run_single(ctx, p, prm) for p in probs]
    lock, r_lock = ctx.optimize_lockstep(probs, prm)
    got, rounds = ctx.optimize_device(probs, prm)
    OD.assert_same(got, ref, (what, "single"))
    OD.assert_same(got, lock, (what, "lockstep"))
    assert rounds == r_lock == max(r["evaluations"] for r in ref)
    return ref


@pytest.mark.parametrize("strict", [True, False])
@pytest.mark.parametrize("which", list(EDGE_SETS))
def test_edges_bitwise(which, strict):
    probs = EDGE_SETS[which]()
    ctx = edge_ctx(strict, probs)
    ref = three_back_ends(ctx, probs, OD.PARAMS, (which, strict))
    assert all(r["evaluations"] > 1 for r in ref)
    ctx.close()


@pytest.mark.parametrize("strict", [True, False])
@pytest.mark.parametrize("res", [1, 64])
def test_penalty_sampling_bitwise(res, strict):
    """integralIntervs 1 and 64 for both penalties; at N = 64 and res 64, 4 160 pose records per problem"""
    probs = [OD.problem(64, 20, 101, dur=2.0), OD.problem(33, 10, 102), OD.problem(5, 10, 103)]
    ctx = edge_ctx(strict, probs, res)
    three_back_ends(ctx, probs, OD.PARAMS, ("res", res, strict))
    ctx.close()


def many_problems(n=1200, seed=7):
    """n problems: N from 2 to 64 (every warp shape), P 0 to 4, durations 1 to 3 s; they finish in different rounds"""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        N = int(rng.choice([2, 3, 5, 8, 16, 31, 32, 33, 47, 64])) if k % 10 else 2 + k % 63
        out.append(OD.problem(N, int(rng.integers(0, 5)), 5000 + k, dur=float(rng.uniform(1.0, 3.0))))
    return out


@pytest.mark.parametrize("strict", [True, False])
def test_thousand_problems_and_slot_reuse(strict):
    probs = many_problems()
    prm = api.default_lbfgs_params(mem_size=16, past=3, delta=1e-6, g_epsilon=0.0, max_iterations=6, min_step=1e-32)
    ctx = edge_ctx(strict, probs)
    ref = [L.run_single(ctx, p, prm) for p in probs]
    ev = [r["evaluations"] for r in ref]
    assert len(set(ev)) >= 3  # problems finish in different rounds
    lock, r_lock = ctx.optimize_lockstep(probs, prm, max_in_flight=len(probs))
    OD.assert_same(lock, ref, ("lockstep", strict))
    assert r_lock == max(ev)
    for m in (1, 7, 64, 0, len(probs)):  # 0: the default, 1 024 slots for 1 200 problems
        got, rounds = ctx.optimize_device(probs, prm, max_in_flight=m)
        OD.assert_same(got, ref, ("device", strict, m))
        if m == 1:
            assert rounds == sum(ev)
        if m == len(probs):
            assert rounds == max(ev)
    ctx.close()
