"""GPU (-m gpu): svsdf_optimize_device — the back end of n problems with its L-BFGS and MINCO on the device gives every problem the bits
of svsdf_optimize and of svsdf_optimize_lockstep on the same context."""
import os
import sys

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_lockstep as L  # noqa: E402  (seeded trajectories, points, contexts and the single-problem reference run)

pytestmark = pytest.mark.gpu
SVSDF_ERR_INVALID = -1
KEYS_INT = ("status", "iterations", "evaluations", "solver_status")
KEYS_BITS = ("x", "T", "coeffs", "cost_at_start", "final_cost")


def problem(N, P, seed, dur=2.5):
    T, co, init_s, final_s, q = L.traj(N, seed, dur)
    x0 = np.r_[api.backward_T(T), q.T.reshape(-1)]
    pts = L.points_near(T, co, P, seed + 1000, spread=2.5) if P else np.zeros((0, 3))
    return dict(N=N, init_s=init_s, final_s=final_s, x0=x0, points=pts)


def mixed_problems(big=True):
    """N = 2, 3, 8, 23, 64; P = 0, 1, tens and (big) one problem above the batched k_outer threshold"""
    out = [problem(2, 0, 11), problem(3, 1, 12), problem(8, 40, 13), problem(23, 70, 14, 1.5), problem(64, 30, 15, 2.0)]
    if big:
        out.append(problem(8, 51000, 16))
    return out


def assert_same(got, ref, what):
    assert len(got) == len(ref)
    for k, (g, r) in enumerate(zip(got, ref)):
        for key in KEYS_INT:
            assert g[key] == r[key], (what, k, key, g[key], r[key])
        for key in KEYS_BITS:
            assert np.array_equal(L.bits(g[key]), L.bits(r[key])), (what, k, key)


PARAMS = api.default_lbfgs_params(mem_size=16, past=3, delta=1e-6, g_epsilon=0.0, max_iterations=0, min_step=1e-32)


@pytest.mark.parametrize("strict", [True, False])
@pytest.mark.parametrize("shape,pp", [("star", (0.0, 0.0, 0.0)), ("star", (0.4, -0.3, 25.0)), ("sdHorseshoe", (0.0, 0.0, 0.0)),
                                      ("Circle", (0.2, 0.1, 10.0)), ("Polygon", (0.0, 0.0, 0.0))])
def test_device_is_bitwise_optimize_and_lockstep(shape, pp, strict):
    ctx = L.ctx_for(shape, pp, strict)
    probs = mixed_problems(big=(shape == "star" and pp[2] == 0.0))
    ref = [L.run_single(ctx, p, PARAMS) for p in probs]
    lock, r_lock = ctx.optimize_lockstep(probs, PARAMS)
    got, rounds = ctx.optimize_device(probs, PARAMS)
    assert_same(got, ref, (shape, pp, strict, "single"))
    assert_same(got, lock, (shape, pp, strict, "lockstep"))
    assert rounds == r_lock == max(r["evaluations"] for r in ref)
    ctx.close()


def test_mesh_and_scale_schedule():
    ctx = L.ctx_for("star_obj_mesh")
    probs = [problem(3, 30, 21), problem(5, 50, 22)]
    prm = api.default_lbfgs_params(max_iterations=6)
    assert_same(ctx.optimize_device(probs, prm)[0], [L.run_single(ctx, p, prm) for p in probs], "mesh")
    ctx.close()
    for strict in (True, False):
        ctx = L.ctx_for("star", strict=strict)
        ctx.set_scale(**api.EXAMPLE_SCALE)
        probs = mixed_problems(big=False)
        assert_same(ctx.optimize_device(probs, PARAMS)[0], [L.run_single(ctx, p, PARAMS) for p in probs], ("scaled", strict))
        ctx.close()


VARIANTS = {
    "max_iterations_0": dict(max_iterations=0), "max_iterations_4": dict(max_iterations=4),
    "nonsmooth_0": dict(nonsmooth_restarts=0), "nonsmooth_8": dict(nonsmooth_restarts=8),
    "mem_1": dict(mem_size=1), "mem_16": dict(mem_size=16), "past_0": dict(past=0), "past_3": dict(past=3),
}


@pytest.mark.parametrize("name", list(VARIANTS))
def test_parameter_variants(name):
    ctx = L.ctx_for("star")
    probs = mixed_problems(big=False)
    prm = api.default_lbfgs_params(**VARIANTS[name])
    ref = [L.run_single(ctx, p, prm) for p in probs]
    got, rounds = ctx.optimize_device(probs, prm)
    assert_same(got, ref, name)
    assert rounds == max(r["evaluations"] for r in ref)
    if name == "max_iterations_4":
        assert any(r["iterations"] == 4 for r in ref)
    ctx.close()


def test_huge_g_epsilon_stops_at_once_and_max_in_flight():
    ctx = L.ctx_for("star")
    probs = mixed_problems(big=False)
    stop = api.default_lbfgs_params(g_epsilon=1e30)
    ref = [L.run_single(ctx, p, stop) for p in probs]
    got, rounds = ctx.optimize_device(probs, stop)
    assert rounds == 1 and all(r["iterations"] == 0 for r in ref)
    assert_same(got, ref, "g_epsilon")
    ref = [L.run_single(ctx, p, PARAMS) for p in probs]
    for m in (1, 3, 0):
        got, rounds = ctx.optimize_device(probs, PARAMS, max_in_flight=m)
        assert_same(got, ref, ("max_in_flight", m))
        if m == 1:
            assert rounds == sum(r["evaluations"] for r in ref)
    ctx.close()


def test_line_search_past_300_s_fails_like_optimize():
    """D = 299.5 s at the start: a step that lengthens the trajectory past 300 s is an invalid evaluation (NaN cost)."""
    ctx = L.ctx_for("star")
    probs = [problem(64, 20, 31, dur=299.5 / 64), problem(3, 20, 32)]
    ref = [L.run_single(ctx, p, PARAMS) for p in probs]
    lock, _ = ctx.optimize_lockstep(probs, PARAMS)
    got, _ = ctx.optimize_device(probs, PARAMS)
    assert_same(got, ref, "300 s")
    assert_same(got, lock, "300 s lockstep")
    ctx.close()


def test_invalid_start_trajectory_ends_with_invalid_and_nan():
    """D = 301 s at the start: the first evaluation is refused (NaN cost), the problem ends with SVSDF_ERR_INVALID; the others run."""
    ctx = L.ctx_for("star")
    probs = [problem(8, 20, 33, dur=301.0 / 8), problem(3, 20, 34)]
    got, _ = ctx.optimize_device(probs, PARAMS)
    assert got[0]["status"] == SVSDF_ERR_INVALID and got[0]["solver_status"] == -1012  # LBFGSERR_INVALID_FUNCVAL
    assert np.isnan(got[0]["final_cost"]) and np.isnan(got[0]["cost_at_start"]) and got[0]["evaluations"] == 1
    assert got[1]["status"] >= 0
    for g, p in zip(got, probs):  # svsdf_optimize (its start cost is not evaluated separately: svsdf_evaluate refuses D >= 300 s)
        ctx.set_points(p["points"])
        rc, x, T, b, st = ctx.optimize(p["init_s"], p["final_s"], p["x0"], p["N"], PARAMS)
        assert g["status"] == rc and (g["iterations"], g["evaluations"], g["solver_status"]) == (st["iterations"], st["evaluations"], st["status"])
        for key, v in (("x", x), ("T", T), ("coeffs", b), ("final_cost", st["final_cost"])):
            assert np.array_equal(L.bits(g[key]), L.bits(v)), key
    assert_same(got, ctx.optimize_lockstep(probs, PARAMS)[0], "301 s lockstep")
    ctx.close()


@pytest.mark.parametrize("over", [dict(mem_size=0), dict(mem_size=-3), dict(past=-1), dict(max_linesearch=0)])
def test_refused_solver_parameters_are_lockstep_results(over):
    """Parameters the L-BFGS refuses: every problem ends at once with the check's code, as in svsdf_optimize_lockstep."""
    ctx = L.ctx_for("star")
    probs = mixed_problems(big=False)
    prm = api.default_lbfgs_params(**over)
    lock, r_lock = ctx.optimize_lockstep(probs, prm)
    got, rounds = ctx.optimize_device(probs, prm)
    assert rounds == r_lock == 0 and all(g["status"] < -1000 for g in got)
    for k, (g, r) in enumerate(zip(got, lock)):
        for key in KEYS_INT:
            assert g[key] == r[key], (over, k, key)
        for key in ("x", "T", "coeffs", "final_cost"):
            assert np.array_equal(L.bits(g[key]), L.bits(r[key])), (over, k, key)
        assert np.isnan(g["cost_at_start"]) and np.isnan(r["cost_at_start"])
    # the context still works afterwards
    ref = [L.run_single(ctx, p, PARAMS) for p in probs[:2]]
    assert_same(ctx.optimize_device(probs[:2], PARAMS)[0], ref, "after refused parameters")
    ctx.close()


def test_context_reuse_cost_grad_bits_and_launches_per_round():
    ctx = L.ctx_for("star")
    probs = mixed_problems(big=False)
    T, co, *_ = L.traj(5, 41)
    pts = L.points_near(T, co, 300, 42)
    ctx.set_points(pts)
    before = ctx.cost_grad(T, co)
    ref = [L.run_single(ctx, p, PARAMS) for p in probs]
    ctx.set_points(pts)
    launches = []
    for sel in ([0, 1, 2, 3, 4], [2], [4, 1, 0, 2, 1, 3], [1, 2]):
        l0 = ctx.kernel_launches()
        got, rounds = ctx.optimize_device([probs[i] for i in sel], PARAMS)
        launches.append((ctx.kernel_launches() - l0 - 1) / rounds)  # one init launch: every problem enters at once
        assert_same(got, [ref[i] for i in sel], sel)
    after = ctx.cost_grad(T, co)
    for a, b in zip(before, after):
        assert np.array_equal(L.bits(a), L.bits(b))
    # per round: blobs, pose table, k_outer (sparse), compaction, k_gsip, finalize, backward — whatever n (rounds where only problems
    # with invalid trajectories run launch fewer; none occur here)
    assert all(x <= 7 for x in launches) and max(launches) == 7, launches
    ctx.close()


def test_errors():
    ctx = L.ctx_for("star")
    p = problem(3, 10, 51)
    with pytest.raises(api.SvsdfError):
        ctx.optimize_device([dict(p, N=1, x0=p["x0"][:1])])
    with pytest.raises(api.SvsdfError):
        ctx.optimize_device([p], max_in_flight=65536)
    lib = api.lib()
    la = (api.LockstepProblem * 1)()
    assert lib.svsdf_optimize_device(ctx.h, la, 1, None, 0, None, None, None) != 0  # null initS / finalS / opt_x
    assert lib.svsdf_optimize_device(ctx.h, None, 1, None, 0, None, None, None) != 0
    assert lib.svsdf_optimize_device(None, None, 0, None, 0, None, None, None) != 0
    ctx.close()


def test_lmbm_context_is_refused(tmp_path):
    import subprocess
    so = str(tmp_path / "liblmbm_standin.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", os.path.join(os.path.dirname(L.GOLD), "cpp", "lmbm_standin.cpp"),
                           "-o", so])
    ctx = L.ctx_for("star")
    ctx.set_lmbm_library(so)
    with pytest.raises(api.SvsdfError):
        ctx.optimize_device([problem(3, 10, 61)])
    ctx.close()
