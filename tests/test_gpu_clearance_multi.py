"""GPU (-m gpu): svsdf_map_clearance_multi — every problem of a mixed batch bit for bit equal to its own svsdf_map_clearance call (N = 1 /
8 / 23 / 64, short and long durations, paths far from every obstacle, the same trajectory twice) over the 16 shapes, Circle and Polygon,
a pre-transform, the star.obj mesh, the scale schedule, both builds, d_max = 0 / 0.7 / 3 / +inf, 2-D maps with the padding bits set and
3-D maps; the strict values against the CPU oracle; launches; non-interference; errors."""
import math

import numpy as np
import pytest

import test_gpu_clearance as tc
from implicit_svsdf_planner_b200 import api
from oracle import clearance_oracle, oracle_py

pytestmark = pytest.mark.gpu
bits = tc.bits


def same(r, s):
    assert np.array_equal(r.ij, s.ij) and np.array_equal(bits(r.xy), bits(s.xy))
    assert np.array_equal(bits(r.sdf), bits(s.sdf)) and np.array_equal(bits(r.tstar), bits(s.tstar))
    assert (r.n_occupied, r.n_evaluated, r.n_within, r.n_colliding, r.argmin) == (s.n_occupied, s.n_evaluated, s.n_within, s.n_colliding,
                                                                                s.argmin)
    assert bits(r.min_sdf) == bits(s.min_sdf)


def mixed_batch():
    """N = 1 / 8 / 23 / 64, short and long D, a path far outside the map (empty band), the same trajectory twice."""
    t8 = tc.traj(8, 31)
    T, co = tc.traj(1, 3)
    far = (T, co + np.eye(1, 18, 0)[0] * 500.0)  # x + 500 m
    return [tc.traj(1, 7), t8, tc.traj(23, 12, 0.4), tc.traj(64, 9, 4.6), far, t8, tc.traj(8, 32, 0.3)]


def map_around(trajs, seed, Z=1, cells=40000):
    """A random map around the paths of the first four problems: (occ [X, Y(, Z)], origin, res), about `cells` columns."""
    pts = np.concatenate([tc.path_xy(t[0], t[1]) for t in trajs[:4]])
    lo, hi = pts.min(axis=0) - 6.0, pts.max(axis=0) + 6.0
    res = float(np.sqrt(np.prod(hi - lo) / cells))
    X, Y = (int(v) for v in np.ceil((hi - lo) / res))
    occ = np.random.default_rng(seed).random((X, Y, Z)) < 0.04 / Z
    return (occ[:, :, 0] if Z == 1 else occ), (float(lo[0]), float(lo[1])), res


def check_batch(ctx, trajs, d_maxes=tc.D_MAX):
    for d_max in d_maxes:
        got = ctx.map_clearance_multi(trajs, d_max)
        assert len(got) == len(trajs)
        for (T, co), r in zip(trajs, got):
            same(r, ctx.map_clearance(T, co, d_max))
    return got


@pytest.mark.parametrize("shape,pp", [(s, (0.0, 0.0, 0.0)) for s in tc.SHAPES16 + ["Circle", "Polygon"]] + [("star", (0.4, -0.3, 25.0))])
def test_multi_equals_single_every_shape(shape, pp):
    ctx = tc.ctx_for(shape, pp)
    trajs = mixed_batch()
    occ, origin, res = map_around(trajs, 5)
    tc.set_map(ctx, occ, origin, res)
    check_batch(ctx, trajs)
    ctx.close()


@pytest.mark.parametrize("strict", [True, False])
def test_multi_equals_single_builds_3d_mesh_scale(strict):
    trajs = mixed_batch()
    ctx = tc.ctx_for("star", strict=strict)
    for Z in (1, 3):
        occ, origin, res = map_around(trajs, 20 + Z, Z=Z)
        tc.set_map(ctx, occ, origin, res)
        got = check_batch(ctx, trajs)
        assert got[4].n_evaluated == got[4].n_occupied  # d_max = +inf: every column, even for the far path
    ctx.set_scale(**api.EXAMPLE_SCALE)
    check_batch(ctx, trajs)
    ctx.close()
    ctx = tc.ctx_for("star_obj_mesh", strict=strict)
    small = [tc.traj(1, 7), tc.traj(2, 8), tc.traj(1, 7)]
    occ, origin, res = map_around(small, 9, cells=6000)
    tc.set_map(ctx, occ, origin, res)
    check_batch(ctx, small)
    ctx.close()


def test_multi_band_edge_polygon_tips():
    """The Polygon bar-tip scene of test_band_bound_is_tight_enough_to_matter: at d_max = 0.67 the listed centres lie 0.007 inside the
    radius bound; a rectangle or band that shrank by 1 % would lose them."""
    ctx = tc.ctx_for("Polygon")
    occ = np.ones((400, 400), dtype=bool)
    tc.set_map(ctx, occ, (-8.0, -8.0), 0.04)
    still = (np.array([1.0]), np.zeros(18))
    moved = (np.array([1.0]), np.eye(1, 18, 0)[0] * 0.37)
    for d_max in (0.0, 0.7, 0.05, 0.67):
        got = check_batch(ctx, [still, moved, still], [d_max])
        assert got[0].n_evaluated < got[0].n_occupied and got[0].n_within > 0
    ctx.close()


@pytest.mark.parametrize("shape", ["star", "Circle"])
def test_multi_strict_values_are_the_oracle(shape):
    ctx = tc.ctx_for(shape)
    trajs = [tc.traj(2, 5), tc.traj(1, 6)]
    occ, origin, res = tc.scene_map(*trajs[0], 21, margin=4.0, cells=3000, density=0.08)
    tc.set_map(ctx, occ, origin, res)
    for d_max in (0.0, 0.7, math.inf):
        got = ctx.map_clearance_multi(trajs, d_max)
        for (T, co), r in zip(trajs, got):
            orc = oracle_py.Oracle(shape, threads=min(8, oracle_py.num_procs()))
            orc.set_traj(T, co)
            tc.assert_same(r, clearance_oracle.clearance(orc, occ, origin, res, d_max))
    ctx.close()


def test_launches_fixed_and_non_interference():
    ctx = tc.ctx_for("star")
    T, co = tc.traj(8, 31)
    rng = np.random.default_rng(3)
    pts = np.c_[rng.uniform(-2, 26, 3000), rng.uniform(-4, 8, 3000), np.zeros(3000)]
    ctx.set_points(pts)
    ctx.cost_grad(T, co)
    ref = ctx.cost_grad(T, co)
    probs = [(T, co, pts), (*tc.traj(4, 2), pts[:700])]
    ctx.cost_grad_multi(probs)
    ref_m = ctx.cost_grad_multi(probs)
    resident = ctx.get_points()
    small = tc.scene_map(T, co, 1, margin=4.0, cells=3000)
    large = tc.scene_map(T, co, 2, margin=60.0, cells=2_000_000, density=0.01)
    counts = []
    for occ, origin, rs in (small, large):
        tc.set_map(ctx, occ, origin, rs)
        single = ctx.map_clearance(T, co, 0.7)
        for n in (1, 10, 300):
            n0 = ctx.kernel_launches()
            got = ctx.map_clearance_multi([(T, co)] * n, 0.7)
            counts.append(ctx.kernel_launches() - n0)
            same(got[0], single)
            same(got[-1], single)
    # count, scan, write, pose table, k_outer_multi (the problems share one schedule here), k_compact_multi, k_gsip_multi
    assert counts == [7] * 6, counts
    # no band: count and scan only; n = 0: nothing
    far = (np.array([1.0]), np.eye(1, 18, 0)[0] * 1e4)
    n0 = ctx.kernel_launches()
    got = ctx.map_clearance_multi([far, far], 0.7)
    assert ctx.kernel_launches() - n0 == 2 and all(r.n_evaluated == 0 and r.n_within == 0 for r in got)
    n0 = ctx.kernel_launches()
    assert ctx.map_clearance_multi([], 0.7) == [] and ctx.kernel_launches() == n0
    after = ctx.cost_grad(T, co)
    for x, y in zip(ref, after):
        assert np.array_equal(bits(x), bits(y))
    for a, b in zip(ref_m, ctx.cost_grad_multi(probs)):
        assert bits(a[0]) == bits(b[0]) and np.array_equal(bits(a[1]), bits(b[1])) and np.array_equal(bits(a[2]), bits(b[2])) and a[3] == b[3]
    assert np.array_equal(bits(resident), bits(ctx.get_points()))
    ctx.close()


def test_errors():
    ctx = tc.ctx_for("star")
    T, co = tc.traj(2, 5)
    with pytest.raises(api.SvsdfError) as e:
        ctx.map_clearance_multi([(T, co)])
    assert "status -3" in str(e.value)  # no map
    occ, origin, res = tc.scene_map(T, co, 4, margin=3.0, cells=2000)
    tc.set_map(ctx, occ, origin, res)
    for d in (-1e-9, math.nan, -math.inf):
        with pytest.raises(api.SvsdfError) as e:
            ctx.map_clearance_multi([(T, co)], d)
        assert "status -1" in str(e.value), d
    for bad in ((np.array([1.0, -1.0]), co), (np.array([1.0, np.nan]), co), (np.array([200.0, 200.0]), co),
                (T, np.where(np.arange(co.size) == 3, np.nan, co)), (np.ones(65), np.zeros(18 * 65))):
        n0 = ctx.kernel_launches()
        with pytest.raises(api.SvsdfError) as e:
            ctx.map_clearance_multi([(T, co), bad, (T, co)])
        assert "status -1" in str(e.value) and "problem 1" in str(e.value)
        assert ctx.kernel_launches() == n0  # refused before any work
    # a path at x ~ 1.7e308 (as in test_gpu_clearance.test_errors): its status is the single call's, the others are listed as usual
    b = np.zeros((6, 3))
    b[0, 0] = b[5, 0] = 1.7e308
    T1, co1 = np.array([1.0]), b.T.reshape(-1).copy()
    got = ctx.map_clearance_multi([(T, co), (T1, co1), (T, co)])
    same(got[0], ctx.map_clearance(T, co))
    same(got[2], got[0])
    ij, xy, sdf, ts = tc.dense_values(ctx, T1, co1, occ, origin, res)
    if np.all(np.isfinite(sdf)):
        same(got[1], ctx.map_clearance(T1, co1))
    else:
        assert isinstance(got[1], api.SvsdfError) and "status -4" in str(got[1])
    ctx.close()
