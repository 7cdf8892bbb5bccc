"""GPU (-m gpu): svsdf_cost_grad_multi and svsdf_optimize_lockstep — n problems per set of launches give every problem the bits of its
single-problem call (svsdf_set_points + svsdf_cost_grad, svsdf_optimize) on the same context."""
import os

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, scenes

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.uint64)


def traj(N, seed, dur=2.5):
    """(T [N], coeffs column-major [18 N], init_s, final_s, q) of a seeded spline; N = 1 is a single quintic built by hand."""
    if N == 1:
        rng = np.random.default_rng(seed)
        b = np.zeros((6, 3))
        b[0] = [rng.uniform(-2, 2), rng.uniform(-2, 2), 0.3]
        b[1] = [1.2, 0.4, 0.2]
        b[2] = [0.05, -0.02, 0.0]
        return np.array([dur]), b.T.reshape(-1).copy(), None, None, None
    init_s, final_s, q, _ = scenes.make_trajectory("star", N=N, seed=seed, start=(0.0, 0.0), goal=(3.0 * N, 4.0))
    T = np.full(N, dur)
    b, _, _, _ = api.minco_forward(init_s, final_s, q, T)
    return T, np.ascontiguousarray(b.T).reshape(-1), init_s, final_s, q


def points_near(T, co, P, seed, spread=4.0):
    """P points scattered around the trajectory (some inside the swept volume)."""
    rng = np.random.default_rng(seed)
    N = T.shape[0]
    b = co.reshape(3, 6 * N).T
    ts = rng.uniform(0, T.sum(), size=P)
    xy = scenes.eval_traj_xy(b, T, ts)[:, :2]
    return np.c_[xy + rng.normal(0, spread, size=(P, 2)), np.zeros(P)]


def single(ctx, T, co, pts):
    ctx.set_points(pts)
    cost, gT, gC = ctx.cost_grad(T, co)
    return cost, gT, gC, int(ctx.cost_grad_device(T, co)[1][-1])


def assert_same(multi, ref, what):
    for k, (m, r) in enumerate(zip(multi, ref)):
        assert bits(m[0]) == bits(r[0]), (what, k, m[0], r[0])
        assert np.array_equal(bits(m[1]), bits(r[1])), (what, k, "gradT")
        assert np.array_equal(bits(m[2]), bits(r[2])), (what, k, "gradC")
        assert m[3] == r[3], (what, k, "n_inside", m[3], r[3])


def mixed_batch():
    """P in {1, 7, 66, 3169, 51000 (batched schedule)}, N in {1, 2, 8, 23, 64 (D = 294 s)}, interior points in every problem."""
    out = []
    for k, (N, P, dur) in enumerate([(1, 1, 2.5), (2, 7, 2.5), (8, 66, 2.5), (23, 3169, 1.5), (64, 200, 4.6), (8, 51000, 2.5)]):
        T, co, *_ = traj(N, 100 + k, dur)
        pts = points_near(T, co, P, 200 + k, spread=3.0 if P > 1 else 0.2)
        out.append((T, co, pts))
    return out



def ctx_for(shape, pp=(0.0, 0.0, 0.0), strict=True):
    if shape == "star_obj_mesh":
        g = np.load(os.path.join(GOLD, "fwn_ref.npz"))
        return api.Context("star", poly_params=pp, strict_fp=strict, mesh=(g["star_V"], g["star_F"]))
    return api.Context(shape, poly_params=pp, strict_fp=strict)


@pytest.mark.parametrize("strict", [True, False])
@pytest.mark.parametrize("shape,pp", [("star", (0.0, 0.0, 0.0)), ("star", (0.4, -0.3, 25.0)), ("sdHorseshoe", (0.0, 0.0, 0.0)),
                                      ("Circle", (0.2, 0.1, 10.0)), ("Polygon", (0.0, 0.0, 0.0))])
def test_cost_grad_multi_is_bitwise_the_single_call(shape, pp, strict):
    ctx = ctx_for(shape, pp, strict)
    probs = mixed_batch()
    before = ctx.kernel_launches()
    multi = ctx.cost_grad_multi(probs)
    # both k_outer schedules occur: pose, sparse and batched k_outer, compaction, k_gsip, finalize
    assert ctx.kernel_launches() - before == 6
    ref = [single(ctx, *p) for p in probs]
    assert sum(r[3] for r in ref) > 0  # interior points occur
    assert_same(multi, ref, (shape, pp, strict))
    ctx.close()


def test_cost_grad_multi_mesh_and_scale():
    """The star.obj mesh functor (small batch: it is slow), and the reference's example scale schedule on the analytic star."""
    ctx = ctx_for("star_obj_mesh")
    probs = [(p[0], p[1], p[2][: min(len(p[2]), 120)]) for p in mixed_batch()[:4]]
    assert_same(ctx.cost_grad_multi(probs), [single(ctx, *p) for p in probs], "mesh")
    ctx.close()
    for strict in (True, False):
        ctx = ctx_for("star", strict=strict)
        ctx.set_scale(**api.EXAMPLE_SCALE)
        probs = mixed_batch()[:5]
        assert_same(ctx.cost_grad_multi(probs), [single(ctx, *p) for p in probs], ("scaled", strict))
        ctx.close()


def test_context_reuse_across_batch_sizes_and_launches_per_round():
    ctx = ctx_for("star")
    probs = mixed_batch()[:4]
    ref = [single(ctx, *p) for p in probs]
    launches = []
    for sel in ([0, 1, 2, 3], [2], [3, 1, 0, 2, 1, 0, 3], [1, 2]):
        before = ctx.kernel_launches()
        got = ctx.cost_grad_multi([probs[i] for i in sel])
        launches.append(ctx.kernel_launches() - before)
        assert_same(got, [ref[i] for i in sel], sel)
        assert_same([single(ctx, *probs[0])], [ref[0]], "single in between")
    # all of these problems take the sparse k_outer schedule: pose, k_outer, compaction, k_gsip, finalize
    assert launches == [5, 5, 5, 5]
    ctx.close()


def opt_problems():
    out = []
    for k, N in enumerate([3, 5, 8]):
        T, co, init_s, final_s, q = traj(N, 300 + k)
        tau = api.backward_T(T)
        x0 = np.r_[tau, q.T.reshape(-1)]
        pts = points_near(T, co, 80 + 40 * k, 400 + k, spread=2.5)
        out.append(dict(N=N, init_s=init_s, final_s=final_s, x0=x0, points=pts))
    # one that stops at once: the start point is already a minimiser for the tolerance used below
    out.append(dict(out[0], x0=out[0]["x0"].copy()))
    return out


def run_single(ctx, p, params):
    ctx.set_points(p["points"])
    ctx.set_boundary(p["init_s"], p["final_s"], p["N"])
    f0, _ = ctx.evaluate(p["x0"])
    rc, x, T, b, st = ctx.optimize(p["init_s"], p["final_s"], p["x0"], p["N"], params)
    return dict(status=rc, x=x, T=T, coeffs=b, cost_at_start=f0, final_cost=st["final_cost"], iterations=st["iterations"],
                evaluations=st["evaluations"], solver_status=st["status"])


@pytest.mark.parametrize("scaled", [False, True])
def test_optimize_lockstep_is_bitwise_optimize(scaled):
    ctx = ctx_for("star")
    if scaled:
        ctx.set_scale(**api.EXAMPLE_SCALE)
    probs = opt_problems()
    params = [api.default_lbfgs_params(mem_size=16, past=3, delta=1e-6, g_epsilon=0.0, max_iterations=m, min_step=1e-32) for m in (0, 4)]
    for pi, prm in enumerate(params):
        ref = [run_single(ctx, p, prm) for p in probs]
        if pi == 1:
            assert all(r["iterations"] <= 4 for r in ref) and any(r["iterations"] == 4 for r in ref)  # max_iterations reached
        for m in (1, 3, 0):
            got, rounds = ctx.optimize_lockstep(probs, prm, max_in_flight=m)
            for k, (g, r) in enumerate(zip(got, ref)):
                for key in ("status", "iterations", "evaluations", "solver_status"):
                    assert g[key] == r[key], (m, k, key, g[key], r[key])
                for key in ("x", "T", "coeffs", "cost_at_start", "final_cost"):
                    assert np.array_equal(bits(g[key]), bits(r[key])), (m, k, key)
            if m == 0:
                assert rounds == max(r["evaluations"] for r in ref)
    # a start that stops at once: g_epsilon so large that the first gradient passes the test
    stop = api.default_lbfgs_params(mem_size=16, past=3, delta=1e-6, g_epsilon=1e30, max_iterations=0, min_step=1e-32)
    ref = [run_single(ctx, p, stop) for p in probs[:2]]
    got, rounds = ctx.optimize_lockstep(probs[:2], stop)
    assert all(r["iterations"] == 0 for r in ref) and rounds == 1
    for g, r in zip(got, ref):
        assert g["status"] == r["status"] and np.array_equal(bits(g["x"]), bits(r["x"]))
    ctx.close()


def test_errors():
    ctx = ctx_for("star")
    T, co, *_ = traj(3, 1)
    pts = points_near(T, co, 10, 1)
    with pytest.raises(api.SvsdfError):
        ctx.cost_grad_multi([(np.full(65, 1.0), np.zeros(18 * 65), pts)])  # N = 65
    with pytest.raises(api.SvsdfError):
        ctx.cost_grad_multi([(T, co, pts), (np.array([1.0, -1.0, 1.0]), co, pts)])  # a non-positive duration
    L = api.lib()
    arr = (api.MultiProblem * 1)()
    assert L.svsdf_cost_grad_multi(ctx.h, 1, None) != 0
    assert L.svsdf_cost_grad_multi(ctx.h, 1, arr) != 0  # null trajectory and outputs
    assert L.svsdf_cost_grad_multi(None, 0, None) != 0
    p = opt_problems()[0]
    with pytest.raises(api.SvsdfError):
        ctx.optimize_lockstep([dict(p, N=1, x0=p["x0"][:1])])
    la = (api.LockstepProblem * 1)()
    assert L.svsdf_optimize_lockstep(ctx.h, la, 1, None, 0, None, None) != 0  # null initS / finalS / opt_x
    bad = (api.LockstepProblem * 1)()
    i_s = api._colmajor33(p["init_s"])
    x = p["x0"].copy()
    bad[0].N, bad[0].initS, bad[0].finalS, bad[0].opt_x, bad[0].P, bad[0].stride = p["N"], api._p(i_s), api._p(i_s), api._p(x), -1, 2
    assert L.svsdf_optimize_lockstep(ctx.h, bad, 1, None, 0, None, None) != 0  # P < 0
    ctx.close()


def test_lmbm_context_is_refused(tmp_path):
    import subprocess
    so = str(tmp_path / "liblmbm_standin.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", os.path.join(os.path.dirname(GOLD), "cpp", "lmbm_standin.cpp"),
                           "-o", so])
    ctx = ctx_for("star")
    ctx.set_lmbm_library(so)
    with pytest.raises(api.SvsdfError):
        ctx.optimize_lockstep(opt_problems()[:1])
    ctx.close()
