"""GPU parity tests (run with -m gpu on an H100): the CUDA path, called through the C ABI (include/svsdf.h via
implicit_svsdf_planner_b200.api), against the CPU oracle on the same seeded inputs and against the committed golden
vectors.

Parity statement (north_star: cost and gradient within 1e-6 relative of the reference):
  * strict build (product default, -fmad=false) vs the oracle's default build: both sides perform the same IEEE
    operations in the same order and use the same published sin/cos algorithm (fdlibm; the oracle's copy is
    oracle/portable_sincos.hpp), so every per-point result of the outer solve — sdf, t*, FD gradient — is BIT-IDENTICAL;
    cost / gradC / gradT differ only by summation order (<= 1e-11 relative); interior (GSIP) points are bitwise too
    (atan2 of the ring direction is the same pinned fdlibm restatement on both sides).
  * versus the oracle built with glibc's sin/cos ("glibc" variant = the reference's actual x86-64 behaviour) the cost
    agrees to 1e-12 and the gradient to ~1e-5: the reference's sign-descent is ill-conditioned where the robot is at
    rest (trajectory ends) and a 1-ulp difference in sin/cos moves t* by ~1e-5 there.  The same happens when the
    reference's own source is compiled with FMA contraction ("fma" variant).  These tests pin that noise floor.
  * strict_fp = 0 (opt-in FMA build of the kernels) sits inside the same noise floor (<= 1e-4).
"""
import os

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, scenes

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

ALL_SHAPES = ["star", "sdHorseshoe", "sdPie", "sdPie2", "sdArc", "sdTunnel", "sdCutDisk", "sdTrapezoid", "sdRhombus",
              "sdHeart", "sdRoundedX", "bigX", "sdRoundedCross", "sdOrientedVesica", "sdMoon", "sdUnevenCapsule",
              "Circle", "unknown_mesh_shape"]


def nrel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def gT_err(gT, gT_ref, gC_ref):
    """Error of gradT in units of its own error budget.  gradT(j) = -sum_{points in pieces > j} G.vel is a heavily
    cancelling sum (sum of |terms| ~ 1e3 * |gradT| on these scenes), so its attainable accuracy is set by the scale of
    the terms, which is the scale of gradC (same G, times beta0 instead of vel): budget = ||gradT|| + 1e-3 ||gradC||."""
    return np.linalg.norm(np.asarray(gT) - gT_ref) / (np.linalg.norm(gT_ref) + 1e-3 * np.linalg.norm(gC_ref))


def pts0(sc):
    return np.c_[sc.points[:, :2], np.zeros(sc.P)]


# ----------------------------------------------------------------------------------------------------------------
# R5: shape functors
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("strict", [False, True])
def test_shape_functors_match_oracle(oracle_mod, strict):
    rng = np.random.default_rng(42)
    rel = np.c_[rng.uniform(-7, 7, size=(5000, 2)), np.zeros(5000)]
    for pp in ((0.0, 0.0, 0.0), (0.6, -0.3, 25.0)):
        for name in ALL_SHAPES:
            ctx = api.Context(name, poly_params=pp, strict_fp=strict)
            s_gpu = ctx.shape_sdf(rel)
            s_cpu = oracle_mod.shape_sdf(name, rel, poly_params=pp)
            assert np.abs(s_gpu - s_cpu).max() <= 1e-12, (name, pp, np.abs(s_gpu - s_cpu).max())
            g_gpu = ctx.shape_grad1(rel)
            g_cpu = oracle_mod.shape_grad1(name, rel, poly_params=pp)
            # FD with dx = 1e-6 amplifies 1-ulp differences by 1e6/2; compare away from SDF creases
            ok = np.abs(g_gpu - g_cpu).max(axis=1) < 1e-6
            assert ok.mean() > 0.995, (name, pp, ok.mean())
            ctx.close()


def test_strict_shape_functors_are_bitwise(oracle_mod):
    """The strict build uses only IEEE-exact operations in the shape functors (+, -, *, sqrt, and divisions either
    native or by Markstein's corrected reciprocal for compile-time divisors), so it must reproduce the CPU bit for bit."""
    rng = np.random.default_rng(77)
    rel = np.c_[rng.uniform(-8, 8, size=(200_000, 2)), np.zeros(200_000)]
    rel[:1000, :2] = rng.uniform(-0.05, 0.05, size=(1000, 2))  # near the origin / symmetry axes
    for pp in ((0.0, 0.0, 0.0), (0.6, -0.3, 25.0)):
        for name in ALL_SHAPES:
            if name == "unknown_mesh_shape":
                continue  # polygon uses atan2 (libm) for its inside test
            ctx = api.Context(name, poly_params=pp, strict_fp=True)
            s_gpu = ctx.shape_sdf(rel)
            s_cpu = oracle_mod.shape_sdf(name, rel, poly_params=pp)
            bad = np.flatnonzero(s_gpu != s_cpu)
            assert bad.size == 0, (name, pp, bad.size, rel[bad[:3]], s_gpu[bad[:3]], s_cpu[bad[:3]])
            ctx.close()


def test_custom_polygon_fallback(oracle_mod):
    poly = [3.0, -1.0, 3.0, 1.0, 0.0, 2.5, -3.0, 1.0, -3.0, -1.0]
    rng = np.random.default_rng(1)
    rel = np.c_[rng.uniform(-6, 6, size=(2000, 2)), np.zeros(2000)]
    ctx = api.Context("custom_poly", polygon=poly)
    assert np.abs(ctx.shape_sdf(rel) - oracle_mod.shape_sdf("custom_poly", rel, polygon=poly)).max() < 1e-12
    g_gpu, g_cpu = ctx.shape_grad1(rel), oracle_mod.shape_grad1("custom_poly", rel, polygon=poly)
    assert (np.abs(g_gpu - g_cpu).max(axis=1) < 1e-9).mean() > 0.995


def test_device_sincos_is_bitwise_the_oracles(oracle_mod):
    rng = np.random.default_rng(8)
    x = np.concatenate([rng.uniform(-10, 10, 400_000), rng.uniform(-1e5, 1e5, 100_000), rng.uniform(-0.8, 0.8, 100_000),
                        [0.0, -0.0, np.pi / 2, np.pi, 1e-300, 0.785398163397448, 0.7853981633974484, 3e5]])
    ctx = api.Context("star", strict_fp=True)
    s_g, c_g = ctx.sincos(x)
    s_c, c_c = oracle_mod.sincos(x)
    assert np.array_equal(s_g, s_c) and np.array_equal(c_g, c_c)
    # and it is an accurate sin/cos: at most 2 ulp away from glibc's
    s_l, c_l = oracle_mod.sincos(x, "glibc")
    assert (np.abs(s_g - s_l) <= 2 * np.spacing(np.abs(s_l))).all() and (np.abs(c_g - c_l) <= 2 * np.spacing(np.abs(c_l))).all()


# ----------------------------------------------------------------------------------------------------------------
# R2: per-point swept-volume SDF queries
# ----------------------------------------------------------------------------------------------------------------
def test_strict_query_is_bit_identical_to_oracle(oracle_mod, scene2k, scene_small_inside):
    for sc in (scene2k, scene_small_inside):
        co = sc.coeffs_colmajor()
        opt = api.TrajOptimizer("star", strict_fp=True)
        sv = opt.sv_manager
        sv.updateTraj(sc.T, co)
        orc = oracle_mod.Oracle("star", threads=oracle_mod.num_procs())
        orc.set_traj(sc.T, co)
        p = pts0(sc)
        s_c, t_c, g_c = orc.query_outer(p)
        s_g, t_g, g_g = sv.getSDFofSweptVolume(p)
        assert np.array_equal(s_g, s_c) and np.array_equal(t_g, t_c) and np.array_equal(g_g, g_c)
        s_c, t_c, g_c, r_c = orc.query(p)
        s_g, t_g, g_g, r_g = sv.getTrueSDFofSweptVolume(p)
        assert np.array_equal(r_c, r_g)  # same GSIP round count for every point
        outside = r_c == 0
        assert np.array_equal(s_g[outside], s_c[outside]) and np.array_equal(t_g[outside], t_c[outside])
        assert np.array_equal(g_g[outside], g_c[outside])
        inside = ~outside
        if inside.any():  # interior (GSIP) branch: same ring samples, same solves, same arg-min -> bitwise as well
            assert np.array_equal(s_g[inside], s_c[inside]) and np.array_equal(t_g[inside], t_c[inside])
            assert np.array_equal(g_g[inside], g_c[inside])  # world-frame unit direction
            assert np.abs(np.linalg.norm(g_g[inside], axis=1) - 1.0).max() < 1e-12


@pytest.mark.parametrize("strict,variant", [(True, "glibc"), (False, "default"), (False, "glibc"), (False, "fma")])
def test_query_agrees_with_other_reference_builds_up_to_flat_minima(oracle_mod, scene2k, scene_small_inside, strict, variant):
    for sc in (scene2k, scene_small_inside):
        co = sc.coeffs_colmajor()
        sv = api.TrajOptimizer("star", strict_fp=strict).sv_manager
        sv.updateTraj(sc.T, co)
        orc = oracle_mod.Oracle("star", threads=oracle_mod.num_procs(), variant=variant)
        orc.set_traj(sc.T, co)
        p = pts0(sc)
        s_c, t_c, g_c, r_c = orc.query(p)
        s_g, t_g, g_g, r_g = sv.getTrueSDFofSweptVolume(p)
        assert np.array_equal(r_c, r_g)
        assert np.abs(s_g - s_c).max() <= 1e-9  # the SDF value is insensitive (second order in t*)
        assert np.median(np.abs(t_g - t_c)) <= 1e-7  # t* is only defined up to the flatness of t -> sdf(t)
        assert (np.abs(g_g - g_c).max(axis=1) < 1e-5).mean() > 0.99


def test_batched_path_is_bit_identical_to_sparse_path(oracle_mod, scene2k, scene_small_inside, monkeypatch):
    """k_outer has two schedules: one point per warp throughout (small problems) and the batched one (choiceTInit, FD
    gradient and chain rule one point per lane, 32 points per warp at a time).  Both must give the oracle's bits."""
    for sc in (scene2k, scene_small_inside):
        co = sc.coeffs_colmajor()
        p = pts0(sc)
        orc = oracle_mod.Oracle("star", threads=oracle_mod.num_procs())
        orc.set_traj(sc.T, co)
        s_c, t_c, g_c, r_c = orc.query(p)
        res = {}
        for mode, grid in (("sparse", None), ("batched", "3"), ("batched-ragged", "7")):
            if grid is None:
                monkeypatch.delenv("SVSDF_FORCE_GRID_OUTER", raising=False)
                monkeypatch.setenv("SVSDF_FORCE_BATCHED", "0")
            else:
                monkeypatch.setenv("SVSDF_FORCE_GRID_OUTER", grid)  # 3 CTAs = 24 warps -> batches of 32 / 16 points per warp
                monkeypatch.setenv("SVSDF_FORCE_BATCHED", "1")
            ctx = api.Context("star")
            s_g, t_g, g_g, r_g = ctx.query(sc.T, co, p)
            out = r_c == 0
            assert np.array_equal(r_g, r_c), mode
            assert np.array_equal(s_g[out], s_c[out]) and np.array_equal(t_g[out], t_c[out]) and np.array_equal(g_g[out], g_c[out]), mode
            ctx.set_points(sc.points)
            res[mode] = ctx.cost_grad(sc.T, co)
        c0, gT0, gC0 = res["sparse"]
        for mode in ("batched", "batched-ragged"):
            c1, gT1, gC1 = res[mode]
            assert abs(c1 - c0) <= 1e-13 * abs(c0) and nrel(gC1, gC0) <= 1e-12 and gT_err(gT1, gT0, gC0) <= 1e-12, mode
    monkeypatch.delenv("SVSDF_FORCE_GRID_OUTER", raising=False)
    monkeypatch.delenv("SVSDF_FORCE_BATCHED", raising=False)


@pytest.mark.parametrize("shape", ALL_SHAPES)
def test_every_shape_through_the_batched_schedule_is_bitwise(oracle_mod, shape, monkeypatch):
    """The batched schedule (layer 1 with exact pruning, quarter-warp descent engine) for every functor, with and without a
    body-frame pre-transform: same bits as the oracle's plain loops."""
    monkeypatch.setenv("SVSDF_FORCE_GRID_OUTER", "2")  # 16 warps -> batches of 25..32 points per warp
    monkeypatch.setenv("SVSDF_FORCE_BATCHED", "1")
    sc = scenes.make_scene("star", 8, 900, clearance=1.6, seed_map=777)
    co = sc.coeffs_colmajor()
    p = pts0(sc)
    for pp in ((0.0, 0.0, 0.0), (0.4, -0.25, 33.0)):
        ctx = api.Context(shape, poly_params=pp)
        orc = oracle_mod.Oracle(shape, poly_params=pp, threads=oracle_mod.num_procs())
        orc.set_traj(sc.T, co)
        s_c, t_c, g_c, r_c = orc.query(p)
        s_g, t_g, g_g, r_g = ctx.query(sc.T, co, p)
        out = r_c == 0
        assert np.array_equal(r_g, r_c), (shape, pp)
        assert np.array_equal(s_g[out], s_c[out]) and np.array_equal(t_g[out], t_c[out]) and np.array_equal(g_g[out], g_c[out]), (shape, pp)
        ctx.close()
    monkeypatch.delenv("SVSDF_FORCE_GRID_OUTER", raising=False)
    monkeypatch.delenv("SVSDF_FORCE_BATCHED", raising=False)


def test_query_matches_committed_golden():
    for name in ("config1_star_2k.npz", "config_inside_400.npz"):
        G = np.load(os.path.join(HERE, "golden", name))
        ctx = api.Context(str(G["shape"]), weight_p=float(G["weight_p"]), safety_hor=float(G["safety_hor"]),
                          rho=float(G["rho"]), strict_fp=True)
        p = np.c_[G["points"][:, :2], np.zeros(G["points"].shape[0])]
        s, t, g, r = ctx.query(G["T"], G["coeffs_colmajor"], p)
        assert np.array_equal(r, G["query_rounds"])
        out = r == 0
        assert np.array_equal(s[out], G["query_sdf"][out]) and np.array_equal(t[out], G["query_tstar"][out])
        assert np.array_equal(g[out], G["query_grad"][out])
        assert np.abs(s - G["query_sdf"]).max() <= 1e-9


# ----------------------------------------------------------------------------------------------------------------
# R1: cost + gradient accumulation
# ----------------------------------------------------------------------------------------------------------------
def test_cost_grad_strict_matches_oracle(oracle_mod, scene2k, scene_small_inside):
    for sc in (scene2k, scene_small_inside):
        co = sc.coeffs_colmajor()
        opt = api.TrajOptimizer("star", weight_p=sc.weight_p, safety_hor=sc.safety_hor, rho=sc.rho, strict_fp=True)
        opt.parallel_points = sc.points
        orc = oracle_mod.Oracle("star", threads=oracle_mod.num_procs())
        orc.set_points(sc.points)
        c0, gT0, gC0, _, inside = orc.cost_grad(sc.T, co)
        c1, gT1, gC1 = opt.addSaftyPenaOnSweptVolumeParallelTrueSDF(sc.T, co)
        assert abs(c1 - c0) <= 1e-12 * abs(c0)
        assert nrel(gC1, gC0) <= 1e-9 and gT_err(gT1, gT0, gC0) <= 1e-9, (nrel(gC1, gC0), gT_err(gT1, gT0, gC0))
        # and against the reference's real libm (glibc): inside the reference's own noise floor
        o_gl = oracle_mod.Oracle("star", threads=oracle_mod.num_procs(), variant="glibc")
        o_gl.set_points(sc.points)
        c2, gT2, gC2, _, _ = o_gl.cost_grad(sc.T, co)
        assert abs(c1 - c2) <= 1e-9 * abs(c2)
        assert nrel(gC1, gC2) <= 1e-4 and gT_err(gT1, gT2, gC2) <= 1e-4


def test_cost_grad_fma_build_stays_within_the_reference_noise_floor(oracle_mod, scene2k, scene_small_inside):
    """strict_fp = 0 lets nvcc contract a*b+c into FMAs.  Cost and per-point SDF still agree to rounding, but the
    gradient inherits the reference algorithm's own sensitivity to contraction (next test): it agrees with the
    un-fused oracle AND with the FMA-compiled oracle only to ~1e-5 (each compiler contracts different pairs)."""
    for sc in (scene2k, scene_small_inside):
        co = sc.coeffs_colmajor()
        opt = api.TrajOptimizer("star", strict_fp=False)
        opt.parallel_points = sc.points
        c1, gT1, gC1 = opt.addSaftyPenaOnSweptVolumeParallelTrueSDF(sc.T, co)
        for variant in ("default", "glibc", "fma"):
            o = oracle_mod.Oracle("star", threads=oracle_mod.num_procs(), variant=variant)
            o.set_points(sc.points)
            c0, gT0, gC0, _, _ = o.cost_grad(sc.T, co)
            assert abs(c1 - c0) <= 1e-9 * abs(c0)
            assert nrel(gC1, gC0) <= 1e-4 and gT_err(gT1, gT0, gC0) <= 1e-4, (variant, nrel(gC1, gC0))


def test_reference_algorithm_is_sensitive_to_fma_contraction(oracle_mod, scene2k):
    """Documents the noise floor: the reference's own algorithm, compiled from the same source with and without FMA
    contraction, disagrees with itself in gradC by ~1e-5 on config 1 while the cost agrees to 1e-15."""
    sc = scene2k
    co = sc.coeffs_colmajor()
    a = oracle_mod.Oracle("star", threads=oracle_mod.num_procs(), variant="glibc")
    b = oracle_mod.Oracle("star", threads=oracle_mod.num_procs(), variant="fma")
    a.set_points(sc.points)
    b.set_points(sc.points)
    ca, gTa, gCa, ppa, _ = a.cost_grad(sc.T, co, per_point=True)
    cb, gTb, gCb, ppb, _ = b.cost_grad(sc.T, co, per_point=True)
    assert abs(ca - cb) <= 1e-12 * abs(ca)
    assert nrel(gCb, gCa) < 1e-4
    # the disagreement comes from a handful of points whose minimiser sits in the flat end of the trajectory
    dt = np.abs(ppa[:, 1] - ppb[:, 1])
    worst = np.argsort(-dt)[:5]
    assert np.all(ppa[worst, 1] > sc.T.sum() - 0.01) or np.all(ppa[worst, 1] < 0.01)


def test_cost_grad_accumulates_and_is_bitwise_deterministic(scene2k):
    sc = scene2k
    co = sc.coeffs_colmajor()
    ctx = api.Context("star")
    ctx.set_points(sc.points)
    c1, gT1, gC1 = ctx.cost_grad(sc.T, co)
    c2, gT2, gC2 = ctx.cost_grad(sc.T, co)
    assert c1 == c2 and np.array_equal(gT1, gT2) and np.array_equal(gC1, gC2)
    rng = np.random.default_rng(0)
    aT, aC = rng.normal(size=sc.N), rng.normal(size=18 * sc.N)
    c3, gT3, gC3 = ctx.cost_grad(sc.T, co, cost0=7.0, gradT0=aT, gradC0=aC)
    assert c3 == c1 + 7.0 and np.array_equal(gT3, gT1 + aT) and np.array_equal(gC3, gC1 + aC)
    # a second context (fresh buffers) gives the same bits
    ctx2 = api.Context("star")
    ctx2.set_points(sc.points)
    c4, gT4, gC4 = ctx2.cost_grad(sc.T, co)
    assert c4 == c1 and np.array_equal(gC4, gC1)


def test_cost_grad_matches_committed_golden():
    for name in ("config1_star_2k.npz", "config_inside_400.npz"):
        G = np.load(os.path.join(HERE, "golden", name))
        ctx = api.Context(str(G["shape"]), weight_p=float(G["weight_p"]), safety_hor=float(G["safety_hor"]),
                          rho=float(G["rho"]), strict_fp=True)
        ctx.set_points(G["points"])
        c, gT, gC = ctx.cost_grad(G["T"], G["coeffs_colmajor"])
        assert abs(c - float(G["cost"])) <= 1e-12 * abs(c)
        assert nrel(gC, G["gradC"]) <= 1e-9 and gT_err(gT, G["gradT"], G["gradC"]) <= 1e-9
        ctx.set_boundary(G["init_s"], G["final_s"], int(G["N"]))
        f, g = ctx.evaluate(G["x0"])
        assert abs(f - float(G["eval_f"])) <= 1e-12 * abs(f)
        assert nrel(g, G["eval_g"]) <= 1e-8


@pytest.mark.parametrize("shape,N", [("sdHorseshoe", 16), ("sdPie", 8), ("sdTunnel", 5), ("sdRoundedCross", 8),
                                     ("sdMoon", 8), ("unknown_mesh_shape", 8)])
def test_other_shapes_and_piece_counts(oracle_mod, shape, N):
    sc = scenes.make_scene(shape if shape in scenes.START_GOAL else "star", N, 600, clearance=2.0)
    co = sc.coeffs_colmajor()
    ctx = api.Context(shape, strict_fp=True)
    ctx.set_points(sc.points)
    orc = oracle_mod.Oracle(shape, threads=oracle_mod.num_procs())
    orc.set_points(sc.points)
    c0, gT0, gC0, pp, inside = orc.cost_grad(sc.T, co, per_point=True)
    c1, gT1, gC1 = ctx.cost_grad(sc.T, co)
    assert c0 > 0
    assert abs(c1 - c0) <= 1e-9 * abs(c0), (shape, c1, c0)
    assert nrel(gC1, gC0) <= 1e-8 and gT_err(gT1, gT0, gC0) <= 1e-8, (shape, nrel(gC1, gC0), gT_err(gT1, gT0, gC0))


@pytest.mark.parametrize("shape", ALL_SHAPES)
def test_every_registry_shape_end_to_end(oracle_mod, shape):
    """Every key of the reference's shapeConstructors registry (+ Circle and the Polygon fallback) through the whole path:
    per-point query bit-identical outside the swept volume, cost / gradient to summation order."""
    sc = scenes.make_scene("star", 8, 240, clearance=1.6, seed_map=4242)
    co = sc.coeffs_colmajor()
    ctx = api.Context(shape)
    orc = oracle_mod.Oracle(shape, threads=oracle_mod.num_procs())
    p = pts0(sc)
    orc.set_traj(sc.T, co)
    s_c, t_c, g_c, r_c = orc.query(p)
    s_g, t_g, g_g, r_g = ctx.query(sc.T, co, p)
    out = r_c == 0
    assert np.array_equal(r_g, r_c)
    assert np.array_equal(s_g[out], s_c[out]) and np.array_equal(t_g[out], t_c[out]) and np.array_equal(g_g[out], g_c[out])
    assert np.abs(s_g - s_c).max() <= 1e-9
    ctx.set_points(sc.points)
    orc.set_points(sc.points)
    c0, gT0, gC0, _, _ = orc.cost_grad(sc.T, co)
    c1, gT1, gC1 = ctx.cost_grad(sc.T, co)
    assert abs(c1 - c0) <= 1e-12 * max(1.0, abs(c0)) and nrel(gC1, gC0) <= 1e-8 and gT_err(gT1, gT0, gC0) <= 1e-8


def test_body_frame_offset_of_the_shape(oracle_mod):
    sc = scenes.make_scene("star", 8, 500, clearance=2.6)
    co = sc.coeffs_colmajor()
    pp = (0.4, -0.2, 20.0)
    ctx = api.Context("star", poly_params=pp, strict_fp=True)
    ctx.set_points(sc.points)
    orc = oracle_mod.Oracle("star", poly_params=pp, threads=oracle_mod.num_procs())
    orc.set_points(sc.points)
    c0, gT0, gC0, _, _ = orc.cost_grad(sc.T, co)
    c1, gT1, gC1 = ctx.cost_grad(sc.T, co)
    assert abs(c1 - c0) <= 1e-12 * abs(c0) and nrel(gC1, gC0) <= 1e-8


# ----------------------------------------------------------------------------------------------------------------
# R3 / R4: full cost callback and host optimiser
# ----------------------------------------------------------------------------------------------------------------
def test_evaluate_callback_matches_oracle(oracle_mod, scene2k):
    sc = scene2k
    opt = api.TrajOptimizer("star", weight_p=sc.weight_p, safety_hor=sc.safety_hor, rho=sc.rho, strict_fp=True)
    opt.parallel_points = sc.points
    opt.setConditions(sc.init_s, sc.final_s, sc.N)
    orc = oracle_mod.Oracle("star", threads=oracle_mod.num_procs())
    orc.set_points(sc.points)
    orc.set_conditions(sc.init_s, sc.final_s, sc.N)
    rng = np.random.default_rng(4)
    for k in range(3):
        x = sc.x0 + (0.05 * k) * rng.normal(size=sc.x0.size)
        f0, g0 = orc.evaluate(x)
        f1, g1 = opt.costFunction(x)
        assert abs(f1 - f0) <= 1e-12 * abs(f0)
        assert nrel(g1, g0) <= 1e-8, nrel(g1, g0)
        assert np.abs(opt.ctx.last_costs() - orc.last_costs()).max() <= 1e-8 * abs(f0)


def test_optimize_reduces_cost_and_final_point_agrees_with_oracle(oracle_mod):
    sc = scenes.make_scene("star", 8, 1500, clearance=2.9)
    opt = api.TrajOptimizer("star", weight_p=sc.weight_p, safety_hor=sc.safety_hor, rho=sc.rho, strict_fp=True)
    opt.parallel_points = sc.points
    opt.setConditions(sc.init_s, sc.final_s, sc.N)
    f_start, _ = opt.costFunction(sc.x0)
    params = api.default_lbfgs_params(mem_size=16, past=3, delta=1e-5, g_epsilon=0.0, max_iterations=40, min_step=1e-32)
    rc, x, T, b, st = opt.optimize_traj(sc.init_s, sc.final_s, sc.x0, sc.N, params)
    assert st["final_cost"] < f_start and st["iterations"] >= 3 and st["evaluations"] >= st["iterations"]
    assert np.all(T > 0) and np.all(np.isfinite(b))
    # final cost and gradient on identical inputs (the optimiser's final x) within 1e-6 of the oracle
    orc = oracle_mod.Oracle("star", threads=oracle_mod.num_procs())
    orc.set_points(sc.points)
    orc.set_conditions(sc.init_s, sc.final_s, sc.N)
    f0, g0 = orc.evaluate(x)
    f1, g1 = opt.costFunction(x)
    assert abs(f1 - f0) <= 1e-12 * abs(f0) and nrel(g1, g0) <= 1e-8
    if st["status"] >= 0:  # on a line-search failure lbfgs_ref.hpp:541-547 restores x but reports the last trial's f
        assert abs(st["final_cost"] - f1) <= 1e-9 * abs(f1)


def test_replay_of_the_reference_lmbm_trace():
    """tests/golden/lmbm_trace_star_400.npz holds iterates visited by the reference's OWN outer solver (the prebuilt LMBM
    binary with its default parameters) while minimising the oracle's cost callback.  The CUDA callback must return the
    same cost and gradient at each of them — so plugging svsdf_evaluate into lmbm_optimize retraces the reference run."""
    G = np.load(os.path.join(HERE, "golden", "lmbm_trace_star_400.npz"))
    opt = api.TrajOptimizer(str(G["shape"]), weight_p=float(G["weight_p"]), safety_hor=float(G["safety_hor"]), rho=float(G["rho"]))
    opt.parallel_points = G["points"]
    opt.setConditions(G["init_s"], G["final_s"], int(G["N"]))
    assert G["xs"].shape[0] >= 30 and float(G["final_f"]) < 0.6 * float(G["fs"][0])  # LMBM made real progress
    for x, f0, g0 in zip(G["xs"], G["fs"], G["gs"]):
        f1, g1 = opt.costFunction(x)
        assert abs(f1 - f0) <= 1e-11 * abs(f0), (f1, f0)
        assert nrel(g1, g0) <= 1e-7, nrel(g1, g0)


def test_progress_callback_can_cancel(scene2k):
    sc = scene2k
    opt = api.TrajOptimizer("star")
    opt.parallel_points = sc.points[:500]
    calls = []

    def progress(_user, _x, k):
        calls.append(k)
        return 1 if k >= 2 else 0

    rc, x, T, b, st = opt.optimize_traj(sc.init_s, sc.final_s, sc.x0, sc.N, api.default_lbfgs_params(max_iterations=50), progress)
    assert calls == [1, 2] and st["status"] == 2 and rc == 2  # LBFGS_CANCELED


# ----------------------------------------------------------------------------------------------------------------
# Edge cases and error behaviour
# ----------------------------------------------------------------------------------------------------------------
def test_edge_cases(oracle_mod, scene2k):
    sc = scene2k
    co = sc.coeffs_colmajor()
    ctx = api.Context("star", strict_fp=True)
    # empty query set
    ctx.set_points(np.zeros((0, 3)))
    c, gT, gC = ctx.cost_grad(sc.T, co)
    assert c == 0.0 and not gT.any() and not gC.any()
    s, t, g, r = ctx.query(sc.T, co, np.zeros((0, 3)))
    assert s.size == 0
    # one point; duplicated points act as integer weights (SURVEY.md A.10)
    one = sc.points[[np.argmin(np.abs(sc.points[:, 0] - 12.0))]]
    ctx.set_points(one)
    c1, gT1, gC1 = ctx.cost_grad(sc.T, co)
    ctx.set_points(np.repeat(one, 3, axis=0))
    c3, gT3, gC3 = ctx.cost_grad(sc.T, co)
    assert abs(c3 - 3 * c1) <= 1e-12 * max(1.0, abs(c3)) and np.allclose(gC3, 3 * gC1, rtol=1e-12, atol=1e-12)
    # far away points: no penalty at all
    far = sc.points.copy()
    far[:, 1] += 1000.0
    ctx.set_points(far)
    c, gT, gC = ctx.cost_grad(sc.T, co)
    assert c == 0.0 and not gT.any() and not gC.any()
    # stride-2 input equals stride-3 input; z is ignored
    ctx.set_points(sc.points[:100, :2])
    a = ctx.cost_grad(sc.T, co)
    zz = sc.points[:100].copy()
    zz[:, 2] = 123.0
    ctx.set_points(zz)
    b = ctx.cost_grad(sc.T, co)
    assert a[0] == b[0] and np.array_equal(a[2], b[2])
    # minimal and larger piece counts
    for N in (2, 3, 32):
        scn = scenes.make_scene("star", N, 200, clearance=2.6)
        ctx.set_points(scn.points)
        orc = oracle_mod.Oracle("star", threads=oracle_mod.num_procs())
        orc.set_points(scn.points)
        c0, gT0, gC0, _, _ = orc.cost_grad(scn.T, scn.coeffs_colmajor())
        c1, gT1, gC1 = ctx.cost_grad(scn.T, scn.coeffs_colmajor())
        assert abs(c1 - c0) <= 1e-12 * max(1.0, abs(c0)) and nrel(gC1, gC0) <= 1e-8, (N, c1, c0)


def test_errors_are_reported_not_thrown(scene2k):
    sc = scene2k
    co = sc.coeffs_colmajor()
    ctx = api.Context("star")
    with pytest.raises(api.SvsdfError):  # points not set
        ctx.cost_grad(sc.T, co)
    ctx.set_points(sc.points[:10])
    with pytest.raises(api.SvsdfError):  # too many pieces
        ctx.cost_grad(np.full(65, 1.0), np.zeros(18 * 65))
    with pytest.raises(api.SvsdfError):  # total duration >= 300 s (sw_manager.hpp:380)
        ctx.cost_grad(sc.T * 20.0, co)
    bad = sc.T.copy()
    bad[2] = -1.0
    with pytest.raises(api.SvsdfError):
        ctx.cost_grad(bad, co)
    with pytest.raises(api.SvsdfError):  # evaluate without boundary conditions
        ctx.evaluate(sc.x0)
    # the context still works afterwards
    c, _, _ = ctx.cost_grad(sc.T, co)
    assert np.isfinite(c)


# ----------------------------------------------------------------------------------------------------------------
# Full-size (BASELINE config 2: 200k points) size-independent properties
# ----------------------------------------------------------------------------------------------------------------
def _full_size_check(oracle_mod, shape, N, P, mesh=None, spot=1500, cost_evals=True, scene_shape=None, polygon=None):
    """Size-independent properties at a BASELINE config's full size + a spot check of the FULL-SIZE run's per-point outputs
    (batched schedule) against the oracle."""
    sc = scenes.make_scene(scene_shape or (shape if shape in scenes.START_GOAL else "star"), N, P)
    co = sc.coeffs_colmajor()
    ctx = api.Context(shape, mesh=mesh, polygon=polygon)
    ctx.set_points(sc.points)
    c, gT, gC = ctx.cost_grad(sc.T, co)
    assert np.isfinite(c) and c > 0
    if cost_evals:
        # additivity over a partition of the query set
        half = sc.P // 2
        ctx.set_points(sc.points[:half])
        ca, gTa, gCa = ctx.cost_grad(sc.T, co)
        ctx.set_points(sc.points[half:])
        cb, gTb, gCb = ctx.cost_grad(sc.T, co)
        assert abs((ca + cb) - c) <= 1e-11 * c and nrel(gCa + gCb, gC) <= 1e-11 and gT_err(gTa + gTb, gT, gC) <= 1e-11
        # permutation invariance
        perm = np.random.default_rng(3).permutation(sc.P)
        ctx.set_points(sc.points[perm])
        cp, gTp, gCp = ctx.cost_grad(sc.T, co)
        assert abs(cp - c) <= 1e-11 * c and nrel(gCp, gC) <= 1e-11
    # per-point outputs of the full-size run (this is the batched schedule) on a random subset vs the oracle: bitwise outside
    # the swept volume, round counts equal, interior values to 1e-9
    p_all = np.c_[sc.points[:, :2], np.zeros(sc.P)]
    s_g, t_g, g_g, r_g = ctx.query(sc.T, co, p_all)
    idx = np.sort(np.random.default_rng(5).choice(sc.P, size=spot, replace=False))
    orc = oracle_mod.Oracle(shape, threads=oracle_mod.num_procs(), mesh=mesh, polygon=polygon)
    orc.set_traj(sc.T, co)
    s_c, t_c, g_c, r_c = orc.query(p_all[idx])
    out = r_c == 0
    assert np.array_equal(r_g[idx], r_c)
    assert np.array_equal(s_g[idx][out], s_c[out]) and np.array_equal(t_g[idx][out], t_c[out]) and np.array_equal(g_g[idx][out], g_c[out])
    assert np.abs(s_g[idx] - s_c).max() <= 1e-9
    # and the subset's share of the cost through the reduction
    sub = sc.points[idx]
    orc.set_points(sub)
    c0, gT0, gC0, _, _ = orc.cost_grad(sc.T, co)
    ctx.set_points(sub)
    c1, gT1, gC1 = ctx.cost_grad(sc.T, co)
    assert abs(c1 - c0) <= 1e-12 * max(abs(c0), 1.0) and nrel(gC1, gC0) <= 1e-8
    ctx.close()


def test_full_size_properties_200k(oracle_mod):
    """BASELINE config 2: star, N = 8, 200 000 points."""
    _full_size_check(oracle_mod, "star", 8, 200_000)


def test_full_size_properties_config3_500k(oracle_mod):
    """BASELINE config 3: sdHorseshoe (concave), N = 16, 500 000 points."""
    _full_size_check(oracle_mod, "sdHorseshoe", 16, 500_000)


def test_full_size_properties_config4_polygon_500k(oracle_mod):
    """BASELINE config 4 as this release of the reference runs it: the outline of shapes/star.obj (40 vertices) through the Polygon
    fallback functor, N = 16, 500 000 points (the crossing test's sign filter against the oracle's two atan2 per edge)."""
    import json

    xy = np.array(json.load(open(os.path.join(HERE, "golden", "obj_outlines.json")))["star"]["outline_xy"])
    poly = xy[np.argsort(np.arctan2(xy[:, 1], xy[:, 0]))].reshape(-1)
    _full_size_check(oracle_mod, "star_obj_outline_polygon", 16, 500_000, scene_shape="sdHorseshoe", polygon=poly)


def test_full_size_properties_config4m_mesh_500k(oracle_mod):
    """BASELINE config 4 through the triangle-mesh functor (getonlySDF_igl): the reference's shapes/star.obj (152 v / 300 f),
    N = 16, 500 000 points — the float winding-number hierarchy and the pruned closest-triangle search at full size."""
    g = np.load(os.path.join(HERE, "golden", "fwn_ref.npz"))
    _full_size_check(oracle_mod, "star_obj_mesh_sdf", 16, 500_000, mesh=(g["star_V"], g["star_F"]), scene_shape="sdHorseshoe", spot=800)
