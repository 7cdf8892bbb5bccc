"""Deformable robots at the limits of their inputs on the H100: the scaled kernels (k_outer_scaled / k_gsip_scaled and their
multi-problem forms, strict build unless stated) on the edge trajectories under edge schedules, against the reference's own
code (tests/golden/ref_pin_scale_edges.npz; the pairs and what each reaches: tests/golden/make_scale_edges_golden.py and
tests/test_oracle_scale_edges.py) and the scaled oracle, per point and bit for bit, under every schedule hook; single points
through cost_grad against the oracle's cost_grad; whole scenes against the summation-order restatement (tests/reduction_ref.py);
cost_grad_multi and optimize_device on a scaled context; the FMA build; the device sin/cos where the schedule's arguments end;
the zero-phase schedule against the rigid kernels; the schedules svsdf_set_scale refuses."""
import os
import sys

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)
import make_scale_edges_golden as mke  # noqa: E402
import reduction_ref as R  # noqa: E402
import test_gpu_lockstep as L  # noqa: E402
import test_oracle_scale_edges as E  # noqa: E402  (the CPU side: fixture access, hard sin arguments, refused schedules)
from oracle import scale_py  # noqa: E402

pytestmark = pytest.mark.gpu
HOOK_VARS = ("SVSDF_FORCE_BATCHED", "SVSDF_FORCE_GRID_OUTER", "SVSDF_FORCE_GSIP_WIDE", "SVSDF_FORCE_GRID_GSIP",
             "SVSDF_FORCE_POSE_WINDOWS", "SVSDF_FORCE_OUTER_CHUNK")
# the k_outer hooks of tests/test_gpu_outer_edges.py, both k_gsip variants and a one-CTA k_gsip grid, the three pose-window
# modes and outer chunks of 1 to 4 (each read at svsdf_create); every pair of the fixture runs under each, one at a time
HOOKS = {
    "default": {}, "sparse": {"SVSDF_FORCE_BATCHED": "0"},
    "sparse_grid1": {"SVSDF_FORCE_BATCHED": "0", "SVSDF_FORCE_GRID_OUTER": "1"},
    "batched_grid1": {"SVSDF_FORCE_BATCHED": "1", "SVSDF_FORCE_GRID_OUTER": "1"},
    "batched_grid3": {"SVSDF_FORCE_BATCHED": "1", "SVSDF_FORCE_GRID_OUTER": "3"},
    "batched_grid7": {"SVSDF_FORCE_BATCHED": "1", "SVSDF_FORCE_GRID_OUTER": "7"},
    "gsip8": {"SVSDF_FORCE_GSIP_WIDE": "0"}, "gsip22": {"SVSDF_FORCE_GSIP_WIDE": "1"},
    "gsip22_grid1": {"SVSDF_FORCE_GSIP_WIDE": "1", "SVSDF_FORCE_GRID_GSIP": "1"},
}
# the pose windows serve the batched seed scan and the chunk groups the batched descent pass: both run on the batched schedule
HOOKS.update({f"pose{k}_batched": {"SVSDF_FORCE_POSE_WINDOWS": str(k), "SVSDF_FORCE_BATCHED": "1", "SVSDF_FORCE_GRID_OUTER": "3"}
              for k in (0, 1, 2)})
HOOKS.update({f"chunk{k}_batched_grid1": {"SVSDF_FORCE_OUTER_CHUNK": str(k), "SVSDF_FORCE_BATCHED": "1",
                                          "SVSDF_FORCE_GRID_OUTER": "1"} for k in (1, 2, 3, 4)})


def _hooks(monkeypatch, hook="default"):
    for v in HOOK_VARS:
        monkeypatch.delenv(v, raising=False)
    for k, v in HOOKS[hook].items():
        monkeypatch.setenv(k, v)


def _sched(sk):
    v = mke.SCHEDULES[sk]
    return dict(a=v[0:2], b=v[2:4], w=v[4:6], phi=v[6:8])


def _ctx(shape, sk=None, strict=True):
    ctx = api.Context(shape, strict_fp=strict)
    if sk is not None:
        ctx.set_scale(**_sched(sk))
    return ctx


def _assert_bits(got, want, what):
    for a, b, n in zip(got, want, ("sdf", "t*", "gradient", "rounds")):
        d = E.bits_differ(a, b)
        assert d == 0, (what, n, d)


@pytest.fixture(scope="module")
def gedge():
    return np.load(os.path.join(HERE, "golden", "ref_pin_scale_edges.npz"))


@pytest.fixture(scope="module")
def orefs(oracle_mod, gedge):
    """The scaled oracle's query (with the GSIP round count) and outer solve per pair."""
    out = {}
    for name, sk in mke.pairs():
        orc = E.scaled_oracle(oracle_mod, gedge, name, sk)
        pts = E.inputs(gedge, name)[3]
        out[name, sk] = (orc.query(pts), orc.query_outer(pts))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# per point, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hook", list(HOOKS))
def test_every_pair_is_bitwise_the_reference_and_the_oracle(gedge, orefs, monkeypatch, hook):
    _hooks(monkeypatch, hook)
    for name, sk in mke.pairs():
        shape, T, co, pts = E.inputs(gedge, name)
        ctx = _ctx(shape, sk)
        got = ctx.query(T, co, pts)
        key = f"{name}_{sk}_portable"
        _assert_bits(got[:3], (gedge[key + "_sdf"], gedge[key + "_tstar"], gedge[key + "_grad"]), (name, sk, hook))
        _assert_bits(got, orefs[name, sk][0], (name, sk, hook, "oracle"))
        so, to, go, _ = ctx.query(T, co, pts, outer_only=True)
        _assert_bits((so, to, go), (gedge[key + "_osdf"], gedge[key + "_otstar"], gedge[key + "_ograd"]), (name, sk, hook, "outer"))
        assert np.all(np.isfinite(got[0])) and np.all(np.isfinite(got[2])), (name, sk, hook)
        ctx.close()


def test_zero_phase_is_the_rigid_kernels(gedge, monkeypatch):
    _hooks(monkeypatch)
    for name in mke.MATRIX:
        if "zero_phase" not in mke.MATRIX[name]:
            continue
        shape, T, co, pts = E.inputs(gedge, name)
        rigid, scaled = _ctx(shape), _ctx(shape, "zero_phase")
        _assert_bits(scaled.query(T, co, pts), rigid.query(T, co, pts), name)
        rigid.set_points(pts)
        scaled.set_points(pts)
        for a, b in zip(scaled.cost_grad(T, co), rigid.cost_grad(T, co)):
            assert E.bits_differ(a, b) == 0, name
        rigid.close()
        scaled.close()


# ---------------------------------------------------------------------------------------------------------------------
# the reduction
# ---------------------------------------------------------------------------------------------------------------------
def test_single_points_through_cost_grad_are_bitwise_the_oracle(gedge, orefs, monkeypatch):
    """One point: no summation order.  Outside points with a penalty and interior points of every pair, cost, gradC and gradT
    equal the scaled oracle's cost_grad bits (+-0 equal, as in tests/test_gpu_outer_edges.py)."""
    _hooks(monkeypatch)
    n_out = n_in = 0
    for name, sk in mke.pairs():
        shape, T, co, pts = E.inputs(gedge, name)
        (sdf, _, _, rounds), (so, _, _) = orefs[name, sk]
        picks = list(np.flatnonzero((so > 0) & (sdf < 0.7))[:2]) + list(np.flatnonzero(rounds > 0)[:2])
        orc = scale_py.ScaledOracle(shape, sched=mke.SCHEDULES[sk], threads=1)
        ctx = _ctx(shape, sk)
        for k in picks:
            orc.set_points(pts[k:k + 1])
            ctx.set_points(pts[k:k + 1])
            c0, gT0, gC0, _, _ = orc.cost_grad(T, co)
            c1, gT1, gC1 = ctx.cost_grad(T, co)
            d = sum(E.bits_differ(np.asarray(a) + 0.0, np.asarray(b) + 0.0) for a, b in ((c1, c0), (gC1, gC0), (gT1, gT0)))
            assert d == 0, (name, sk, k, c1, c0)
            n_in += int(rounds[k] > 0)
            n_out += int(rounds[k] == 0)
        ctx.close()
    assert n_out >= 40 and n_in >= 40, (n_out, n_in)


def test_whole_scenes_are_the_summation_order_restatement(gedge, monkeypatch):
    """cost, gradC and gradT of every pair's whole point set: the kernels' summation order restated bit for bit from the query
    (tests/reduction_ref.py with scale=), and within gamma_h of the exactly rounded sums."""
    _hooks(monkeypatch)
    for name, sk in mke.pairs():
        shape, T, co, pts = E.inputs(gedge, name)
        ctx = _ctx(shape, sk)
        sdf, ts, g, rounds = ctx.query(T, co, pts)
        tr = R.point_terms(pts, T, co, sdf, ts, g, 60.0, 0.7, scale=_sched(sk))
        ctx.set_points(pts)
        _, out = ctx.cost_grad_device(T, co)
        c, gT, gC = ctx.cost_grad(T, co)
        grid = max(1, -(-len(pts) // 8))
        ref, info = R.ordered_record(tr, rounds > 0, grid)
        assert R.bits_equal(out, ref), (name, sk, info)
        assert R.bits_equal(np.r_[c, gC, gT], 0.0 + ref[:-1]), (name, sk)
        ex, ab = R.exact_record(tr)
        assert (np.abs(out[:-1] - ex) <= R.gamma_bound(info, ab, len(T))).all(), (name, sk)
        assert np.all(np.isfinite(out)), (name, sk)
        ctx.close()


def test_cost_grad_multi_gives_every_problem_its_single_call_bits(gedge, monkeypatch):
    """One scaled context, the star trajectories of the matrix as one batch (N = 1 ... 64, D up to 299.84 s, interior points in
    several problems), under two schedules: every problem equals set_points + cost_grad on the same context."""
    _hooks(monkeypatch)
    names = [n for n in mke.MATRIX if str(gedge[f"{n}_shape"]) == "star"]
    for sk in ("limit_w", "thin", "example"):
        ctx = _ctx("star", sk)
        probs = [E.inputs(gedge, n)[1:] for n in names]
        multi = ctx.cost_grad_multi(probs)
        ref = []
        for T, co, pts in probs:
            ctx.set_points(pts)
            c, gT, gC = ctx.cost_grad(T, co)
            ref.append((c, gT, gC))
        for k, (m, r) in enumerate(zip(multi, ref)):
            assert E.bits_differ(m[0], r[0]) + E.bits_differ(m[1], r[1]) + E.bits_differ(m[2], r[2]) == 0, (sk, names[k])
        assert sum(m[3] > 0 for m in multi) >= 3, (sk, [m[3] for m in multi])
        assert max(len(p[0]) for p in probs) == 64 and min(len(p[0]) for p in probs) == 1
        ctx.close()


@pytest.mark.parametrize("sk", ["thin", "limit_w"])
def test_optimize_device_is_bitwise_optimize(monkeypatch, sk):
    _hooks(monkeypatch)
    import test_gpu_optimize_device as O

    ctx = L.ctx_for("star")
    ctx.set_scale(**_sched(sk))
    probs = O.mixed_problems(big=False)
    O.assert_same(ctx.optimize_device(probs, O.PARAMS)[0], [L.run_single(ctx, p, O.PARAMS) for p in probs], sk)
    ctx.close()


@pytest.mark.parametrize("name,sk", [("long64", "limit_w"), ("parked", "fast"), ("endpoints", "thin")])
def test_fma_build_stays_within_the_noise_floor(oracle_mod, gedge, monkeypatch, name, sk):
    """strict_fp = 0: the bounds of tests/test_gpu_scale.py's FMA test, and finite."""
    _hooks(monkeypatch)
    shape, T, co, pts = E.inputs(gedge, name)
    orc = scale_py.ScaledOracle(shape, sched=mke.SCHEDULES[sk], threads=min(8, oracle_mod.num_procs()))
    orc.set_points(pts)
    c0, _, gC0, _, _ = orc.cost_grad(T, co)
    ctx = _ctx(shape, sk, strict=False)
    ctx.set_points(pts)
    c1, gT1, gC1 = ctx.cost_grad(T, co)
    ctx.close()
    assert np.isfinite(c1) and np.all(np.isfinite(gC1)) and np.all(np.isfinite(gT1))
    assert abs(c1 - c0) <= 1e-6 * max(1.0, abs(c0)), (c1, c0)
    assert np.linalg.norm(np.asarray(gC1) - gC0) <= 1e-6 * max(1.0, np.linalg.norm(gC0))


# ---------------------------------------------------------------------------------------------------------------------
# the pinned sin/cos below 1e6 and the refused schedules
# ---------------------------------------------------------------------------------------------------------------------
def test_device_sincos_below_1e6_is_bitwise_the_oracles(oracle_mod):
    rng = np.random.default_rng(72)
    hard = E.hard_arguments(2000)
    x = np.concatenate([rng.uniform(1e5, 1e6, 100_000), hard, -hard, [1e5, np.nextafter(1e6, 0), 999999.5]])
    ctx = api.Context("star", strict_fp=True)
    s_g, c_g = ctx.sincos(x)
    s_c, c_c = oracle_mod.sincos(x)
    assert E.bits_differ(s_g, s_c) == 0 and E.bits_differ(c_g, c_c) == 0
    ctx.close()


@pytest.mark.parametrize("bad", E.REFUSED, ids=lambda d: ",".join(f"{k}={v}" for k, v in d.items()))
def test_refused_schedules_keep_the_previous_setting(gedge, monkeypatch, bad):
    """svsdf_set_scale refuses every schedule whose St^-1 is not finite and non-zero somewhere, and keeps the previous one."""
    _hooks(monkeypatch)
    shape, T, co, pts = E.inputs(gedge, "tiny_n2")
    ctx = _ctx(shape, "thin")
    with pytest.raises(api.SvsdfError):
        ctx.set_scale(**bad)
    _assert_bits(ctx.query(T, co, pts)[:3], (gedge["tiny_n2_thin_portable_sdf"], gedge["tiny_n2_thin_portable_tstar"],
                                             gedge["tiny_n2_thin_portable_grad"]), bad)
    ctx.close()


@pytest.mark.parametrize("ok", E.ACCEPTED, ids=lambda d: ",".join(f"{k}={v}" for k, v in d.items()))
def test_accepted_limits_give_finite_outputs(gedge, monkeypatch, ok):
    """Each side of the bounds that svsdf_set_scale accepts: every query output and the cost finite."""
    _hooks(monkeypatch)
    shape, T, co, pts = E.inputs(gedge, "endpoints")
    ctx = _ctx(shape)
    ctx.set_scale(**ok, w=(0.0, 0.3))
    sdf, ts, g, _ = ctx.query(T, co, pts)
    ctx.set_points(pts)
    c, gT, gC = ctx.cost_grad(T, co)
    assert all(np.all(np.isfinite(a)) for a in (sdf, ts, g, c, gT, gC)), ok
    ctx.close()
