"""GPU tests of the cost path's last stage (run with -m gpu on an H100): point_contribution, the per-warp accumulators of
outer_body, the interior slots of gsip_body, finalize_body and k_finalize_multi — entry by entry.

The reference is tests/reduction_ref.py, fed with svsdf_query's per-point outputs on the same context (every input of
point_contribution is one of them):
  * strict build: every record (svsdf_cost_grad, svsdf_cost_grad_device, each problem of svsdf_cost_grad_multi) equals the
    kernels' summation order restated (ordered_record) BIT FOR BIT, and every entry lies within gamma_h * sum |terms| of its
    exactly rounded sum (exact_record), h the longest addition chain of the schedule;
  * FMA build (strict_fp = 0): every entry within gamma_h * sum |terms| + KAPPA * u * sum B of the exactly rounded sum of the
    terms restated from the FMA context's own query outputs (B: each term's magnitude bound), which removes the t* noise
    floor the oracle comparison has at flat minima.
The grid is what the runtime picks: ceil(P / 8) CTAs while that is below one full wave (P <= 8 * SMs), otherwise
SVSDF_FORCE_GRID_OUTER, or, for the production call, the one candidate among SMs x {1, 2, 3, 4} whose restated order matches.
"""
import os
import sys

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, scenes

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
sys.path.insert(0, HERE)
sys.path.insert(0, GOLD)
import make_outer_edges_golden as mko  # noqa: E402
import reduction_ref as R  # noqa: E402

# The FMA build's allowance per term, in units of u * B.  Each term is at most about 30 roundings deep in either build
# (pos / vel: 12, sin / cos of yaw, the rotation: 3, rg: 4, the smoothedL1 band: 5, d, w and the yaw term: 7, G, gdT: 5,
# beta: 3, the product: 1) and B bounds every intermediate magnitude, so the strict and the contracted evaluation each lie
# within about 30 u B of the real value: 60 u B apart; the two builds' sin / cos differ by a few ulp more (in B's 1 + |yaw|).
KAPPA = 64.0


def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def pts3(p):
    p = np.atleast_2d(np.asarray(p, dtype=np.float64))
    return np.c_[p[:, :2], np.zeros(len(p))]


def make_ctx(monkeypatch, shape="star", grid=None, batched=None, wide=None, scale=None, **kw):
    """A context created under the schedule hooks (read once at svsdf_create)."""
    for var, val in (("SVSDF_FORCE_GRID_OUTER", grid), ("SVSDF_FORCE_BATCHED", batched), ("SVSDF_FORCE_GSIP_WIDE", wide)):
        if val is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, str(int(val)))
    if shape == "star_obj_mesh":
        g = np.load(os.path.join(GOLD, "fwn_ref.npz"))
        ctx = api.Context("star", mesh=(g["star_V"], g["star_F"]), **kw)
    else:
        ctx = api.Context(shape, **kw)
    for var in ("SVSDF_FORCE_GRID_OUTER", "SVSDF_FORCE_BATCHED", "SVSDF_FORCE_GSIP_WIDE"):
        monkeypatch.delenv(var, raising=False)
    if scale is not None:
        ctx.set_scale(**scale)
    return ctx


def terms_of(ctx, T, co, pts, weight_p, safety_hor, scale=None):
    """The terms and the interior flag.  A point takes the interior branch when its OUTER solve gives sdf <= 0; the query then
    reports the branch's depth -r*, which can be > 0 (r* < 0), so the flag is the round count, not the sign of the result."""
    sdf, ts, g, rounds = ctx.query(T, co, pts3(pts))
    return R.point_terms(pts, T, co, sdf, ts, g, weight_p, safety_hor, scale=scale), rounds > 0


def check_strict(ctx, T, co, pts, weight_p, safety_hor, grid=None, batched=None, scale=None):
    """Both single-problem calls against the restated order (bits) and the exactly rounded sums (gamma_h)."""
    P = len(pts)
    if grid is None:
        assert P <= 8 * sm_count()  # one partial wave: the runtime's grid is ceil(P / 8)
        grid = max(1, -(-P // 8))
    tr, inside = terms_of(ctx, T, co, pts, weight_p, safety_hor, scale)
    ctx.set_points(pts3(pts))
    _, out = ctx.cost_grad_device(T, co)
    c, gT, gC = ctx.cost_grad(T, co)
    ref, info = R.ordered_record(tr, inside, grid, batched)
    N = len(T)
    assert R.bits_equal(out, ref), (info, np.flatnonzero(out.view(np.int64) != ref.view(np.int64))[:8])
    assert R.bits_equal(np.r_[c, gC, gT], 0.0 + ref[:-1])
    ex, ab = R.exact_record(tr)
    assert (np.abs(out[:-1] - ex) <= R.gamma_bound(info, ab, N)).all()
    return tr, inside, out, info


SC = {}


def scene(name):
    if name not in SC:
        if name == "scene2k":
            SC[name] = scenes.make_scene("star", 8, 2000)
        elif name == "small_inside":
            SC[name] = scenes.make_scene("star", 8, 400, clearance=2.35)
        elif name == "config2":
            SC[name] = scenes.make_scene("star", 8, 200_000)
    return SC[name]


def active_first(ctx, sc, seed=0):
    """The scene's points, the ones with a penalty (active outside or interior) first, in a seeded order."""
    tr, inside = terms_of(ctx, sc.T, sc.coeffs_colmajor(), sc.points, sc.weight_p, sc.safety_hor)
    perm = np.random.default_rng(seed).permutation(sc.P)
    hot = (tr.active | inside)[perm]
    return sc.points[np.r_[perm[hot], perm[~hot]]]


def path_points(sc, n, jitter, seed):
    b = sc.coeffs_colmajor().reshape(3, -1).T
    xy = scenes.eval_traj_xy(b, sc.T, np.linspace(0.0, float(sc.T.sum()), n))[:, :2]
    return xy + np.random.default_rng(seed).uniform(-jitter, jitter, xy.shape)


# ---------------------------------------------------------------------------------------------------------------------
# strict build: bit for bit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [0, 1, 31, 32, 33, 257])
def test_small_point_counts(monkeypatch, P):
    sc = scene("small_inside")
    ctx = make_ctx(monkeypatch, weight_p=sc.weight_p, safety_hor=sc.safety_hor)
    pts = active_first(ctx, sc)[:P]
    tr, inside, out, _ = check_strict(ctx, sc.T, sc.coeffs_colmajor(), pts, sc.weight_p, sc.safety_hor)
    if P == 0:
        assert R.bits_equal(out, np.zeros(1 + 19 * sc.N + 1))
    else:
        assert tr.active.any()
    if P >= 33:
        assert inside.any() and (tr.active & ~inside).any()


@pytest.mark.parametrize("P", [383, 384])
def test_batched_threshold_at_a_forced_grid(monkeypatch, P):
    """P = 128 g - 1 runs the sparse schedule and P = 128 g the batched one on g = 3 CTAs (the runtime's rule, not forced)."""
    sc = scene("scene2k")
    ctx = make_ctx(monkeypatch, grid=3, weight_p=sc.weight_p, safety_hor=sc.safety_hor)
    pts = active_first(ctx, sc, seed=1)[:P]
    _, _, _, info = check_strict(ctx, sc.T, sc.coeffs_colmajor(), pts, sc.weight_p, sc.safety_hor, grid=3)
    assert info["batched"] == (P == 384)


@pytest.mark.parametrize("grid", [1, 3, 37, 396])
def test_forced_batched_schedule(monkeypatch, grid):
    sc = scene("scene2k")
    ctx = make_ctx(monkeypatch, grid=grid, batched=1, weight_p=sc.weight_p, safety_hor=sc.safety_hor)
    check_strict(ctx, sc.T, sc.coeffs_colmajor(), sc.points, sc.weight_p, sc.safety_hor, grid=grid, batched=True)


@pytest.mark.parametrize("name", ["tiny_k1", "long64", "parked", "junction", "broken"])
def test_outer_edge_scenes(monkeypatch, name):
    """N = 1 (gradT exactly [0.0]), N = 64 with D = 299.84 s (19 N + 1 = 1217 accumulators, 153 finalize CTAs), a parked
    trajectory, t* exactly on a junction and t* = D past the last piece's subtraction chain."""
    shape, T, co, pts = mko.scene(name)
    pts = pts[:1000]
    N = len(T)
    sh = 8.0 if name == "junction" else 0.7  # the junction's points lie a few metres from the path
    ctx = make_ctx(monkeypatch, shape, safety_hor=sh)
    tr, inside, out, _ = check_strict(ctx, T, co, pts, 60.0, sh)
    if N == 1:
        assert R.bits_equal(out[1 + 18:1 + 19], [0.0])
    assert tr.active.any()
    if name == "long64":
        assert len(np.unique(tr.piece[tr.active])) > 32


def test_all_points_beyond_the_horizon_give_exact_zeros(monkeypatch):
    shape, T, co, pts = mko.scene("far")
    ctx = make_ctx(monkeypatch, shape)
    tr, _, out, _ = check_strict(ctx, T, co, pts, 60.0, 0.7)
    assert not tr.active.any() and R.bits_equal(out, np.zeros(1 + 19 * len(T) + 1))


def test_all_points_interior(monkeypatch):
    sc = scene("scene2k")
    ctx = make_ctx(monkeypatch, weight_p=sc.weight_p, safety_hor=sc.safety_hor)
    pts = path_points(sc, 300, 0.05, 3)
    tr, inside, out, _ = check_strict(ctx, sc.T, sc.coeffs_colmajor(), pts, sc.weight_p, sc.safety_hor)
    assert inside.all() and out[-1] == 300.0


@pytest.mark.parametrize("n_path,grid", [(60, None), (1500, 188)])
def test_many_interior_points_over_many_pieces(monkeypatch, n_path, grid):
    """More interior slots than one lane stride (> 32) and than a CTA's threads (> 1024), spread over all 8 pieces: the piece
    matching of finalize_body's interior loops."""
    sc = scene("small_inside")
    ctx = make_ctx(monkeypatch, grid=grid, weight_p=sc.weight_p, safety_hor=sc.safety_hor)
    pts = np.r_[path_points(sc, n_path, 0.3, 4), sc.points[:200, :2]]
    pts = pts[np.random.default_rng(5).permutation(len(pts))]
    tr, inside, _, _ = check_strict(ctx, sc.T, sc.coeffs_colmajor(), pts, sc.weight_p, sc.safety_hor, grid=grid)
    assert inside.sum() > (1024 if n_path > 1024 else 32)
    assert len(np.unique(tr.piece[inside])) == sc.N


@pytest.mark.parametrize("offset", [0.0, 0.005, 0.01])
def test_penalty_edges(monkeypatch, offset):
    """safety_hor made from one point's sdf: x = safety_hor - sdf exactly 0 (inactive), in the smoothing band, at its edge."""
    sc = scene("small_inside")
    probe = make_ctx(monkeypatch)
    sdf, _, _, _ = probe.query(sc.T, sc.coeffs_colmajor(), pts3(sc.points))
    k = int(np.argmin(np.abs(sdf - 0.5)))
    sh = float(sdf[k]) + offset
    ctx = make_ctx(monkeypatch, weight_p=sc.weight_p, safety_hor=sh)
    tr, _, _, _ = check_strict(ctx, sc.T, sc.coeffs_colmajor(), sc.points, sc.weight_p, sh)
    x = sh - sdf[k]
    assert tr.active[k] == (x > 0)
    if offset == 0.0:
        assert x == 0.0 and not tr.active[k]
    elif offset == 0.005:
        assert 0.0 < x < 0.01


@pytest.mark.parametrize("case", ["pretransform", "Polygon", "star_obj_mesh", "scaled", "scaled_pretransform"])
def test_functors_and_the_scaled_chain_rule(monkeypatch, case):
    sc = scene("small_inside")
    shape = {"Polygon": "Polygon", "star_obj_mesh": "star_obj_mesh"}.get(case, "star")
    pp = (0.4, -0.25, 33.0) if "pretransform" in case else (0.0, 0.0, 0.0)
    scale = api.EXAMPLE_SCALE if "scaled" in case else None
    ctx = make_ctx(monkeypatch, shape, scale=scale, poly_params=pp, weight_p=sc.weight_p, safety_hor=sc.safety_hor)
    pts = sc.points if case != "star_obj_mesh" else sc.points[::4]
    tr, _, _, _ = check_strict(ctx, sc.T, sc.coeffs_colmajor(), pts, sc.weight_p, sc.safety_hor, scale=scale)
    assert tr.active.any()


# ---------------------------------------------------------------------------------------------------------------------
# full size
# ---------------------------------------------------------------------------------------------------------------------
def test_config2_three_ways_bit_for_bit():
    """BASELINE config 2 (star, N = 8, 200 000 points, the production grid): set_points with stride 3 (several 16384-point
    chunks, P not a multiple of one), cost_grad and cost_grad_device with 1 and 3 repeats agree bit for bit with each other
    and with the restated order on exactly one candidate grid, and lie within gamma_h of the exactly rounded sums."""
    sc = scene("config2")
    co = sc.coeffs_colmajor()
    ctx = api.Context("star", weight_p=sc.weight_p, safety_hor=sc.safety_hor)
    tr, inside = terms_of(ctx, sc.T, co, sc.points, sc.weight_p, sc.safety_hor)
    ctx.set_points(pts3(sc.points))
    c, gT, gC = ctx.cost_grad(sc.T, co)
    _, out1 = ctx.cost_grad_device(sc.T, co, repeats=1)
    _, out3 = ctx.cost_grad_device(sc.T, co, repeats=3)
    assert R.bits_equal(out1, out3) and R.bits_equal(np.r_[c, gC, gT], 0.0 + out1[:-1])
    hits = []
    for m in (1, 2, 3, 4):
        ref, info = R.ordered_record(tr, inside, m * sm_count())
        if R.bits_equal(out1, ref):
            hits.append(info)
    assert len(hits) == 1, hits
    ex, ab = R.exact_record(tr)
    assert (np.abs(out1[:-1] - ex) <= R.gamma_bound(hits[0], ab, sc.N)).all()
    assert hits[0]["batched"] and inside.any()


def test_config3_500k_within_the_bound():
    sc = scenes.make_scene("sdHorseshoe", 16, 500_000)
    co = sc.coeffs_colmajor()
    ctx = api.Context("sdHorseshoe", weight_p=sc.weight_p, safety_hor=sc.safety_hor)
    tr, inside = terms_of(ctx, sc.T, co, sc.points, sc.weight_p, sc.safety_hor)
    ctx.set_points(sc.points)
    _, out = ctx.cost_grad_device(sc.T, co)
    ex, ab = R.exact_record(tr)
    h = max_chains(tr, inside, [m * sm_count() for m in (1, 2, 3, 4)], sc.N)
    assert (np.abs(out[:-1] - ex) <= R.gamma(h) * ab).all()
    assert out[-1] == inside.sum()


def max_chains(tr, inside, grids, N):
    """The largest h of the candidate grids (an upper bound for whichever the runtime picked)."""
    use = tr.active & ~inside
    h = None
    for g in grids:
        sch = R.warp_schedule(len(use), g, R.is_batched(len(use), g))
        chain = (np.where(sch >= 0, use[np.maximum(sch, 0)], False)).sum(axis=1).max()
        hg = R.chain_lengths(dict(grid=g, n_in=int(inside.sum()), max_chain=int(chain)), N)
        h = hg if h is None else np.maximum(h, hg)
    return h


# ---------------------------------------------------------------------------------------------------------------------
# svsdf_cost_grad_multi: k_outer_multi's virtual grids and k_finalize_multi
# ---------------------------------------------------------------------------------------------------------------------
def test_multi_problem_records_are_the_restated_order(monkeypatch):
    _, T1, co1, p1 = mko.scene("tiny_k1")
    sc = scene("small_inside")
    _, T64, co64, p64 = mko.scene("long64")
    probs = [(T1, co1, p1[:1]), (sc.T, sc.coeffs_colmajor(), sc.points[:300]), (T64, co64, p64[:1000])]
    ctx = make_ctx(monkeypatch, weight_p=sc.weight_p, safety_hor=sc.safety_hor)
    res = ctx.cost_grad_multi(probs)
    n_inside = 0
    for (T, co, pts), (c, gT, gC, ni) in zip(probs, res):
        tr, inside = terms_of(ctx, T, co, pts, sc.weight_p, sc.safety_hor)
        ref, info = R.ordered_record(tr, inside, max(1, -(-len(pts) // 8)))
        assert R.bits_equal(np.r_[c, gC, gT], 0.0 + ref[:-1]) and ni == ref[-1], (len(T), len(pts))
        n_inside += ni
    assert n_inside > 0


# ---------------------------------------------------------------------------------------------------------------------
# FMA build
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["small_inside", "config2"])
def test_fma_build_within_rounding_of_its_own_terms(monkeypatch, name):
    """strict_fp = 0, terms restated from the same context's query (SVSDF_FORCE_GSIP_WIDE fixes the interior variant, so the
    query and the cost evaluation run the same code): |out - exact| <= gamma_h sum |terms| + KAPPA u sum B per entry."""
    sc = scene(name)
    co = sc.coeffs_colmajor()
    ctx = make_ctx(monkeypatch, wide=0, strict_fp=False, weight_p=sc.weight_p, safety_hor=sc.safety_hor)
    tr, inside = terms_of(ctx, sc.T, co, sc.points, sc.weight_p, sc.safety_hor)
    ctx.set_points(sc.points)
    _, out = ctx.cost_grad_device(sc.T, co)
    ex, ab = R.exact_record(tr)
    bsum = R.bound_sum(tr)
    grids = [max(1, -(-sc.P // 8))] if sc.P <= 8 * sm_count() else [m * sm_count() for m in (1, 2, 3, 4)]
    h = max_chains(tr, inside, grids, sc.N)
    err = np.abs(out[:-1] - ex)
    bound = R.gamma(h) * ab * (1.0 + 1e-12) + KAPPA * R.U * bsum
    assert (err <= bound).all(), np.max(err / np.maximum(bound, 1e-300))
    assert out[-1] == inside.sum()
    scale = np.maximum(np.abs(ex), 1e-300)
    print(f"\nFMA build {name}: max |out - exact| / |exact| = {np.max(np.where(ex != 0, err / scale, 0.0)):.3e}, "
          f"max err / bound = {np.max(err / np.maximum(bound, 1e-300)):.3e}")
