"""Deformable robots on the H100: the scaled kernels (k_outer_scaled / k_gsip_scaled, strict build) against the reference's
own code (tests/golden/ref_pin_scale.npz) and the scaled oracle (oracle/scale_py.py), per point and bit for bit, in both k_outer schedules and both
k_gsip variants; the identity schedule against the rigid kernels; the optimiser; the FMA build; the error cases."""
import os
import sys

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, scenes

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_scale_golden as mks  # noqa: E402
from oracle import scale_py  # noqa: E402

pytestmark = pytest.mark.gpu

# k_outer schedule x k_gsip variant (test hooks read at svsdf_create)
MODES = {
    "sparse_gsip8": {"SVSDF_FORCE_BATCHED": "0", "SVSDF_FORCE_GSIP_WIDE": "0"},
    "batched_gsip22": {"SVSDF_FORCE_BATCHED": "1", "SVSDF_FORCE_GRID_OUTER": "2", "SVSDF_FORCE_GSIP_WIDE": "1"},
}
HOOKS = ("SVSDF_FORCE_BATCHED", "SVSDF_FORCE_GRID_OUTER", "SVSDF_FORCE_GSIP_WIDE", "SVSDF_FORCE_GRID_GSIP")


def _hooks(monkeypatch, mode=None):
    for v in HOOKS:
        monkeypatch.delenv(v, raising=False)
    for k, v in (MODES[mode] if mode else {}).items():
        monkeypatch.setenv(k, v)


def _sched(sk):
    v = mks.SCHEDULES[sk]
    return dict(a=v[0:2], b=v[2:4], w=v[4:6], phi=v[6:8])


def _bits_equal(a, b):
    a = np.ascontiguousarray(a, dtype=np.float64).ravel()
    b = np.ascontiguousarray(b, dtype=np.float64).ravel()
    return a.shape == b.shape and bool(np.all(a.view(np.int64) == b.view(np.int64)))


def _ctx(shape, pp=(0.0, 0.0, 0.0), strict=True, mesh=None, params=(60.0, 0.7, 3.8)):
    wp, sh, rho = params
    return api.Context(shape, poly_params=pp, weight_p=wp, safety_hor=sh, rho=rho, strict_fp=strict, mesh=mesh)


@pytest.fixture(scope="module")
def gscale():
    return np.load(os.path.join(HERE, "golden", "ref_pin_scale.npz"))


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("sk", ["example", "aniso"])
def test_every_shape_is_bitwise_the_reference_code(gscale, monkeypatch, sk, mode):
    _hooks(monkeypatch, mode)
    g = gscale
    T, co, pts = g["T"], g["coeffs"], g["points"]
    pts0 = np.c_[pts, np.zeros(len(pts))]
    n_in = 0
    for ip, pp in enumerate(mks.PRE):
        for s in mks.SHAPES:
            ctx = _ctx(s, pp, params=g["params"])
            ctx.set_scale(**_sched(sk))
            sdf, ts, grad, _ = ctx.query(T, co, pts0)
            key = f"portable_{sk}_{ip}_{s}"
            for a, n in ((sdf, "_sdf"), (ts, "_tstar"), (grad, "_grad")):
                b = g[key + n]
                bad = np.flatnonzero((np.asarray(a).view(np.int64) != b.view(np.int64)).reshape(len(b), -1).any(axis=1))
                assert bad.size == 0, (key + n, bad.size, bad[:4], np.asarray(a)[bad[:2]], b[bad[:2]])
            n_in += int((sdf <= 0).sum())
            ctx.close()
    assert n_in >= 100


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("pp", [(0.0, 0.0, 0.0), (0.3, -0.2, 25.0)], ids=["plain", "pre"])
def test_mesh_functor_is_bitwise_the_oracle(oracle_mod, monkeypatch, mode, pp):
    _hooks(monkeypatch, mode)
    m = scenes.extrude_outline(scenes.star_outline(n_per_edge=2), half_height=0.49)
    sc = scenes.make_scene("star", 6, 120, clearance=2.35)
    co = sc.coeffs_colmajor()
    pts0 = np.c_[sc.points[:, :2], np.zeros(sc.P)]
    sched = mks.SCHEDULES["example"]
    orc = scale_py.ScaledOracle(sched=sched, mesh=m, poly_params=pp, threads=min(8, oracle_mod.num_procs()))
    orc.set_traj(sc.T, co)
    ref = orc.query(pts0)
    ctx = _ctx("ignored", pp, mesh=m)
    ctx.set_scale(**_sched("example"))
    got = ctx.query(sc.T, co, pts0)
    for a, b in zip(got[:3], ref[:3]):
        assert _bits_equal(a, b)
    assert int((ref[0] <= 0).sum()) >= 1


@pytest.mark.parametrize("mode", list(MODES))
def test_cost_grad_matches_the_oracle(oracle_mod, gscale, monkeypatch, mode):
    """Single points: cost, gradC and gradT bit for bit; the whole set: the sums to 1e-11 (summation order)."""
    _hooks(monkeypatch, mode)
    g = gscale
    T, co, pts = g["T"], g["coeffs"], g["points"]
    wp, sh, rho = g["params"]
    sched = mks.SCHEDULES["example"]
    orc = scale_py.ScaledOracle("sdPie", sched=sched, weight_p=wp, safety_hor=sh, threads=1)
    orc.set_traj(T, co)
    ctx = _ctx("sdPie", params=g["params"])
    ctx.set_scale(**_sched("example"))
    sdf = orc.query(np.c_[pts, np.zeros(len(pts))])[0]
    picks = list(np.flatnonzero((sdf > 0) & (sdf < sh))[:6]) + list(np.flatnonzero(sdf <= 0)[:4])
    assert len(picks) >= 8
    for k in picks:
        orc.set_points(pts[k:k + 1])
        ctx.set_points(pts[k:k + 1])
        c0, gT0, gC0, _, _ = orc.cost_grad(T, co)
        c1, gT1, gC1 = ctx.cost_grad(T, co)
        assert _bits_equal(c1, c0) and _bits_equal(gC1, gC0) and _bits_equal(gT1, gT0), k
    orc.set_points(pts)
    ctx.set_points(pts)
    c0, gT0, gC0, _, _ = orc.cost_grad(T, co)
    c1, gT1, gC1 = ctx.cost_grad(T, co)
    assert abs(c1 - c0) <= 1e-11 * abs(c0)
    assert np.linalg.norm(np.asarray(gC1) - gC0) <= 1e-11 * np.linalg.norm(gC0)
    assert np.abs(np.asarray(gT1) - gT0).max() <= 1e-11 * np.linalg.norm(gC0)


def test_identity_schedule_and_unset_scale_are_the_rigid_kernels(monkeypatch):
    _hooks(monkeypatch)
    sc = scenes.make_scene("star", 8, 2000)
    co = sc.coeffs_colmajor()
    pts0 = np.c_[sc.points[:, :2], np.zeros(sc.P)]
    rigid = _ctx("star", params=(sc.weight_p, sc.safety_hor, sc.rho))
    r_q = rigid.query(sc.T, co, pts0)
    rigid.set_points(sc.points)
    r_c = rigid.cost_grad(sc.T, co)
    ctx = _ctx("star", params=(sc.weight_p, sc.safety_hor, sc.rho))
    ctx.set_points(sc.points)
    ctx.set_scale(**_sched("identity"))
    for a, b in zip(ctx.query(sc.T, co, pts0), r_q):
        assert _bits_equal(a, b)
    for a, b in zip(ctx.cost_grad(sc.T, co), r_c):
        assert _bits_equal(a, b)
    # a reused context: a real schedule changes the result, set_scale(None) brings the rigid bits back
    ctx.set_scale(**_sched("example"))
    assert not _bits_equal(ctx.query(sc.T, co, pts0)[0], r_q[0])
    ctx.set_scale(None)
    for a, b in zip(ctx.query(sc.T, co, pts0), r_q):
        assert _bits_equal(a, b)
    for a, b in zip(ctx.cost_grad(sc.T, co), r_c):
        assert _bits_equal(a, b)


def test_optimize_with_the_example_schedule_is_deterministic(monkeypatch):
    _hooks(monkeypatch)
    sc = scenes.make_scene("star", 6, 300, clearance=2.6)
    # a budget large enough to end on the relative-decrease test (status >= 0), not on the iteration cap
    params = api.default_lbfgs_params(mem_size=16, past=3, delta=1e-5, g_epsilon=0.0, max_iterations=200, min_step=1e-32)
    runs = []
    for _ in range(2):
        opt = api.TrajOptimizer("star", weight_p=sc.weight_p, safety_hor=sc.safety_hor, rho=sc.rho, strict_fp=True)
        opt.ctx.set_scale(**api.EXAMPLE_SCALE)
        opt.parallel_points = sc.points
        opt.setConditions(sc.init_s, sc.final_s, sc.N)
        f0, _ = opt.costFunction(sc.x0)
        rc, x, T, b, st = opt.optimize_traj(sc.init_s, sc.final_s, sc.x0, sc.N, params)
        assert rc >= 0 and st["final_cost"] < f0 and np.all(T > 0) and np.all(np.isfinite(b))
        runs.append((x, T, b, st["final_cost"]))
    for a, b in zip(*runs):
        assert _bits_equal(a, b)


def test_fma_build_stays_within_the_noise_floor(oracle_mod, gscale, monkeypatch):
    _hooks(monkeypatch)
    g = gscale
    T, co, pts = g["T"], g["coeffs"], g["points"]
    wp, sh, rho = g["params"]
    orc = scale_py.ScaledOracle("star", sched=mks.SCHEDULES["example"], weight_p=wp, safety_hor=sh, threads=1)
    orc.set_points(pts)
    c0, _, gC0, _, _ = orc.cost_grad(T, co)
    ctx = _ctx("star", strict=False, params=g["params"])
    ctx.set_scale(**_sched("example"))
    ctx.set_points(pts)
    c1, _, gC1 = ctx.cost_grad(T, co)
    assert abs(c1 - c0) <= 1e-6 * max(1.0, abs(c0))
    assert np.linalg.norm(np.asarray(gC1) - gC0) <= 1e-6 * max(1.0, np.linalg.norm(gC0))


@pytest.mark.parametrize("bad", [
    dict(a=(0.5, 1.0), b=(0.5, 0.0)),            # a - |b| = 0: S(t) can be singular
    dict(a=(1.0, 0.3), b=(0.0, -0.4)),           # negative b counts by its magnitude
    dict(a=(-1.0, 1.0)),
    dict(a=(float("nan"), 1.0)),
    dict(a=(1.0, 1.0), b=(float("inf"), 0.0)),
    dict(a=(1.0, 1.0), w=(float("nan"), 0.0)),
    dict(a=(1.0, 1.0), phi=(0.0, float("-inf"))),
    dict(a=(1.0, 1.0), b=(0.1, 0.0), w=(1e4, 0.0)),  # sin argument beyond 1e6 rad within 300 s
], ids=lambda d: ",".join(f"{k}={v}" for k, v in d.items()))
def test_invalid_schedules_are_rejected(bad):
    ctx = _ctx("star")
    with pytest.raises(api.SvsdfError):
        ctx.set_scale(**bad)
    with pytest.raises(api.SvsdfError):
        api.scale_matrix(0.0, **bad)
