"""GPU tests of the rigid multi-problem kernels at the limits of their inputs (run with -m gpu on an H100): k_pose_table_multi,
k_outer_multi (both schedules), k_compact_multi, k_gsip_multi and k_finalize_multi, through svsdf_cost_grad_multi and
svsdf_map_clearance_multi, on the edge scenes of the outer solve (tests/golden/make_outer_edges_golden.py) and of the interior
branch (tests/golden/make_gsip_edges_golden.py).

include/svsdf.h promises every problem of a multi call the bits of its own single call, n_inside included, in both builds.  Here:
  * one point per problem: every point of the reference fixtures (ref_pin_outer_edges.npz, ref_pin_gsip_edges.npz, "portable"
    variant) is its own problem, and its record equals the restated order (tests/reduction_ref.py) of the terms built from the
    reference's own sdf, t* and gradient, bit for bit, and its single call;
  * whole scenes as problems of one call, ordered so that k_gsip_multi switches problems A -> B -> A, skips problems without inside
    points and meets P = 0 problems first, in the middle and last, next to a 17 000-point long64 problem that runs the batched
    schedule in the same call;
  * every functor through the multi path; per-point outputs through svsdf_map_clearance_multi against clearance_oracle;
  * n = 65 535 (k_finalize_multi's grid.y limit), n = 65 536 refused, and a sequence of calls on one context whose sizes shrink and
    grow while the k_gsip variant switches.
Each under the schedule hooks (read when a context is created): the production choice, SVSDF_FORCE_BATCHED = 0 / 1 with
SVSDF_FORCE_GRID_OUTER, SVSDF_FORCE_GSIP_WIDE = 0 / 1 and SVSDF_FORCE_GRID_GSIP = 1 (one CTA walks every inside slot, so it reloads
its blob on every problem change).  ±0 count as equal.
"""
import math
import os
import sys
import time

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api
from oracle import clearance_oracle

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
sys.path.insert(0, HERE)
sys.path.insert(0, GOLD)
import make_gsip_edges_golden as mkg  # noqa: E402
import make_outer_edges_golden as mko  # noqa: E402
import reduction_ref as R  # noqa: E402
import test_gpu_clearance as tc  # noqa: E402
import test_gpu_clearance_multi as tcm  # noqa: E402

WEIGHT_P, SAFETY_HOR = 60.0, 3.0  # a horizon of 3 m makes most edge points active (the far scene's never are)
ALL_SHAPES = ["star", "sdHorseshoe", "sdPie", "sdPie2", "sdArc", "sdTunnel", "sdCutDisk", "sdTrapezoid", "sdRhombus",
              "sdHeart", "sdRoundedX", "bigX", "sdRoundedCross", "sdOrientedVesica", "sdMoon", "sdUnevenCapsule",
              "Circle", "unknown_mesh_shape"]
PRE = ((0.0, 0.0, 0.0), (0.4, -0.25, 33.0))
ENV = ("SVSDF_FORCE_BATCHED", "SVSDF_FORCE_GRID_OUTER", "SVSDF_FORCE_GSIP_WIDE", "SVSDF_FORCE_GRID_GSIP", "SVSDF_FORCE_OUTER_CHUNK",
       "SVSDF_FORCE_POSE_WINDOWS")
# hook -> (SVSDF_FORCE_BATCHED, SVSDF_FORCE_GRID_OUTER, SVSDF_FORCE_GSIP_WIDE, SVSDF_FORCE_GRID_GSIP)
HOOKS = {"default": (None, None, None, None), "sparse_grid1": (0, 1, None, None), "batched_grid1": (1, 1, None, None),
         "batched_grid3": (1, 3, None, None), "batched_grid7": (1, 7, None, None), "gsip_8warp": (None, None, 0, None),
         "gsip_wide": (None, None, 1, None), "gsip_grid1": (None, None, None, 1)}
SCHED = dict(HOOKS, sparse=(0, None, None, None))  # plus the sparse schedule on the runtime's grid (the functor cases)
BIG_P = 17_000  # long64 points: above 16 x 132 x 8 = 16 896, the batched schedule on the production grid


def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def make_ctx(monkeypatch, shape, hook="default", strict=True, **kw):
    """A context created under a hook of HOOKS (the hooks are read once, at svsdf_create)."""
    for var, val in zip(ENV, SCHED[hook] + (None, None)):
        if val is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, str(val))
    if shape == "star_obj_mesh":
        g = np.load(os.path.join(GOLD, "fwn_ref.npz"))
        kw = dict(kw, mesh=(g["star_V"], g["star_F"]))
        shape = "star"
    ctx = api.Context(shape, weight_p=WEIGHT_P, safety_hor=SAFETY_HOR, strict_fp=strict, **kw)
    for var in ENV:
        monkeypatch.delenv(var, raising=False)
    return ctx


def forced_plan(hook, P):
    """(grid, batched) of a problem of P <= 8 x SMs points under a hook: the runtime's ceil(P / 8) and its batched rule unless forced."""
    batched, grid = SCHED[hook][:2]
    grid = grid or max(1, -(-P // 8))
    return grid, (R.is_batched(P, grid) if batched is None else bool(batched))


def pts3(p):
    p = np.atleast_2d(np.asarray(p, dtype=np.float64))
    return np.c_[p[:, :2], np.zeros(len(p))]


def rec_of(c, gT, gC, ni):
    return np.r_[c, gC, gT, float(ni)]


def bits_same(a, b):
    """Bitwise equality, -0.0 and +0.0 counted as equal."""
    return R.bits_equal(np.asarray(a, dtype=np.float64) + 0.0, np.asarray(b, dtype=np.float64) + 0.0)


def terms_of(ctx, T, co, pts):
    """The terms and the interior flag from svsdf_query on the same context (test_gpu_reduction.terms_of): a point takes the interior
    branch when its OUTER solve gives sdf <= 0, so the flag is the round count, not the sign of the result."""
    sdf, ts, g, rounds = ctx.query(T, co, pts3(pts))
    return R.point_terms(pts, T, co, sdf, ts, g, WEIGHT_P, SAFETY_HOR), rounds > 0


def single_record(ctx, T, co, pts):
    """set_points + cost_grad, with the interior count of svsdf_query on the same context."""
    ctx.set_points(pts3(pts) if len(pts) else np.zeros((0, 3)))
    c, gT, gC = ctx.cost_grad(T, co)
    ni = int((ctx.query(T, co, pts3(pts))[3] > 0).sum()) if len(pts) else 0
    return rec_of(c, gT, gC, ni)


def launches_of(ctx, fn):
    n0 = ctx.kernel_launches()
    out = fn()
    return out, ctx.kernel_launches() - n0


# ---------------------------------------------------------------------------------------------------------------------
# the fixtures: every point of both reference pins, and long64 points on the pieces the thinned fixture misses
# ---------------------------------------------------------------------------------------------------------------------
class Scene:
    def __init__(self, name, shape, T, co, pts, sdf, tstar, grad, osdf):
        self.name, self.shape, self.T, self.co, self.pts = name, shape, np.asarray(T, float), np.asarray(co, float), pts
        self.sdf, self.tstar, self.grad, self.osdf = sdf, tstar, np.asarray(grad).reshape(-1, 3), osdf
        D = 0.0
        for d in self.T:
            D += d
        self.D = D
        self.inside = osdf <= 0  # getTrueSDFofSweptVolume: `if (argmin_dis > 0) return` on the outer solve

    def terms(self, k):
        return R.point_terms(self.pts[k : k + 1], self.T, self.co, self.sdf[k : k + 1], self.tstar[k : k + 1], self.grad[k : k + 1],
                             WEIGHT_P, SAFETY_HOR)


@pytest.fixture(scope="module")
def pinned(oracle_mod):
    out = {}
    for fname, names in (("ref_pin_outer_edges.npz", mko.SCENES), ("ref_pin_gsip_edges.npz", mkg.SCENES)):
        g = np.load(os.path.join(GOLD, fname))
        for key in names:
            out[key] = Scene(key, str(g[f"{key}_shape"]), g[f"{key}_T"], g[f"{key}_coeffs"], g[f"{key}_points"], g[f"{key}_sdf_portable"],
                             g[f"{key}_tstar_portable"], g[f"{key}_grad_portable"], g[f"{key}_osdf_portable"])
    assert sum(len(s.pts) for s in out.values()) == 1479
    # long64's fixture is thinned to 100 points, none of them outside and active on piece 31: four points per wanted piece from the
    # whole scene, with the oracle's outputs (the oracle is the reference's outer solve bit for bit, tests/test_gpu_outer_edges.py)
    shape, T, co, pts = mko.scene("long64")
    orc = oracle_mod.Oracle(shape, threads=oracle_mod.num_procs())
    orc.set_traj(T, co)
    sdf, ts, grad, _ = orc.query(pts)
    osdf = orc.query_outer(pts)[0]
    piece = R.locate_piece(T, ts)[0]
    pick = []
    for i in (0, 31, 32, 63):
        pick += [int(k) for k in np.flatnonzero((piece == i) & (osdf > 0) & (sdf < SAFETY_HOR))[:4]]
    out["long64_pieces"] = Scene("long64_pieces", shape, T, co, pts[pick], sdf[pick], ts[pick], np.asarray(grad)[pick], osdf[pick])
    return out


def by_shape(scenes):
    shapes = {}
    for s in scenes.values():
        shapes.setdefault(s.shape, []).append(s)
    return shapes


# ---------------------------------------------------------------------------------------------------------------------
# 1. one point per problem, against the reference's own outputs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hook", list(HOOKS))
def test_one_point_per_problem_is_the_reference_code(pinned, monkeypatch, hook):
    """Every fixture point its own problem (one call per robot shape: 1 439 star problems with N = 1 .. 64, D up to 299.84 s and
    K1 = 1 .. 1999, 56 Circle problems).  With one point there is no summation order, so the record is ordered_record of the terms
    of the reference's sdf, t* and gradient, bit for bit, and the problem's own set_points + cost_grad."""
    seen = dict(t0=0, tD=0, pieces64=set(), spin_capped=0, yaw_1e6=0, inside={})
    for shape, group in by_shape(pinned).items():
        ctx = make_ctx(monkeypatch, shape, hook)
        probs = [(s.T, s.co, s.pts[k : k + 1], s, k) for s in group for k in range(len(s.pts))]
        res, launches = launches_of(ctx, lambda: ctx.cost_grad_multi([p[:3] for p in probs]))
        # pose table, one k_outer_multi (every problem has one point: one schedule), compaction, k_gsip_multi, finalize
        assert launches == 5, (hook, shape, launches)
        grid, batched = forced_plan(hook, 1)
        for (T, co, p, s, k), (c, gT, gC, ni) in zip(probs, res):
            tr = s.terms(k)
            ref, _ = R.ordered_record(tr, s.inside[k : k + 1], grid, batched)
            rec = rec_of(c, gT, gC, ni)
            assert bits_same(rec, ref), (hook, s.name, k, rec[:3], ref[:3])
            ctx.set_points(p)
            c1, gT1, gC1 = ctx.cost_grad(T, co)
            assert bits_same(rec[:-1], np.r_[c1, gC1, gT1]), (hook, s.name, k)
            act = bool(tr.active[0])
            seen["t0"] += act and s.tstar[k] == 0.0
            seen["tD"] += act and s.tstar[k] == s.D
            if s.name.startswith("long64") and act and not s.inside[k]:
                seen["pieces64"].add(int(tr.piece[0]))
            seen["spin_capped"] += s.name == "spin" and k < len(mko.SPIN_CAPPED)
            seen["yaw_1e6"] += s.name == "yaw_1e6" and act
            if s.name in mkg.SCENES and s.inside[k]:
                assert ni == 1
                seen["inside"][s.name] = seen["inside"].get(s.name, 0) + 1
        ctx.close()
    assert seen["t0"] >= 10 and seen["tD"] >= 10, seen
    assert {0, 31, 32, 63} <= seen["pieces64"], seen
    assert seen["spin_capped"] == len(mko.SPIN_CAPPED) and seen["yaw_1e6"] >= 10, seen
    assert set(seen["inside"]) == set(mkg.SCENES), seen


# ---------------------------------------------------------------------------------------------------------------------
# 2. whole scenes in one launch
# ---------------------------------------------------------------------------------------------------------------------
def scene_order(pinned, shape, with_big):
    """The problems of one call: (label, T, co, pts).  Problems with inside points alternate with problems without (P = 0, junction,
    far); P = 0 problems come first, in the middle and last; endpoints (Circle: circle_static) appears twice with another problem with
    inside points between them, so the interior slots run A -> B -> A.  with_big: a 17 000-point long64 problem, batched on the
    production grid while the others run the sparse schedule."""
    if shape == "star":
        inner = ["endpoints", "midstop", "endpoints", "tiny_k1", "tiny_k21", "tiny_n2", "long64", "parked", "broken", "yaw_6e3",
                 "yaw_1e6", "spin"]
        if with_big:
            inner.insert(6, "long64_big")
        outer = ["junction", "far"]
    else:
        inner = ["circle_static", "circle_spin", "circle_static"]
        outer = ["far"]
    out = []
    for j in range(len(inner) + 1):
        if j in (0, len(inner) // 2, len(inner)):
            s = pinned[inner[min(j, len(inner) - 1)].replace("_big", "")]
            out.append(("empty", s.T, s.co, np.zeros((0, 3))))
        else:
            s = pinned[outer[j % len(outer)]]
            out.append((s.name, s.T, s.co, s.pts))
        if j == len(inner):
            break
        if inner[j] == "long64_big":
            _, T, co, _ = mko.scene("long64")
            out.append(("long64_big", T, co, mko.long64_points(BIG_P, 70 + BIG_P)))
        else:
            s = pinned[inner[j]]
            out.append((s.name, s.T, s.co, s.pts))
    return out


def restated_matches(tr, inside, P, hook):
    """ordered_record for the problem's grid: the forced one, ceil(P / 8) below one wave, else each candidate SMs x {1 .. 4}."""
    if SCHED[hook][1] is not None or P <= 8 * sm_count():
        grid, batched = forced_plan(hook, P)
        return [R.ordered_record(tr, inside, grid, batched)[0]]
    batched = None if SCHED[hook][0] is None else bool(SCHED[hook][0])
    return [R.ordered_record(tr, inside, m * sm_count(), batched)[0] for m in (1, 2, 3, 4)]


@pytest.mark.parametrize("hook", list(HOOKS))
@pytest.mark.parametrize("strict", [True, False], ids=["strict", "fma"])
def test_whole_scenes_in_one_call(pinned, monkeypatch, hook, strict):
    """Every edge scene with all its fixture points is one problem of one call.  Each record equals the problem's single call on a
    fresh context (both builds; fresh, so that both run the 8-warp k_gsip unless a hook fixes it), and in the strict build the restated
    order of svsdf_query's terms.  The launch count shows both k_outer_multi schedules and the interior branch in one call where the
    hook leaves the schedule to the runtime."""
    with_big = SCHED[hook][1] is None and SCHED[hook][0] is None
    for shape in ("star", "Circle"):
        probs = scene_order(pinned, shape, with_big and shape == "star")
        ctx = make_ctx(monkeypatch, shape, hook, strict)
        res, launches = launches_of(ctx, lambda: ctx.cost_grad_multi([p[1:] for p in probs]))
        ctx.close()
        two = with_big and shape == "star"
        assert launches == (6 if two else 5), (hook, shape, launches)
        has_inside = []
        for (label, T, co, pts), (c, gT, gC, ni) in zip(probs, res):
            rec = rec_of(c, gT, gC, ni)
            fresh = make_ctx(monkeypatch, shape, hook, strict)
            want = single_record(fresh, T, co, pts)
            assert bits_same(rec, want), (hook, strict, label, rec[0], want[0], ni, want[-1])
            if strict:
                tr, inside = terms_of(fresh, T, co, pts)
                hits = [r for r in restated_matches(tr, inside, len(pts), hook) if bits_same(rec, r)]
                assert len(hits) == 1, (hook, label, len(hits))
            fresh.close()
            has_inside.append(ni > 0)
        # I and O alternate, P = 0 first, in the middle and last, the repeated interior scene with an I problem between
        assert has_inside == [k % 2 == 1 for k in range(len(probs))], (hook, shape, has_inside)
        labels = [p[0] for p in probs]
        assert labels[0] == labels[-1] == "empty" and "empty" in labels[2:-2], labels
        rep = "endpoints" if shape == "star" else "circle_static"
        a, b = [k for k, lb in enumerate(labels) if lb == rep][:2]
        assert any(has_inside[k] for k in range(a + 1, b)), labels


# ---------------------------------------------------------------------------------------------------------------------
# 3. every functor through the multi path
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ALL_SHAPES + ["star_obj_mesh"])
def test_every_shape_on_the_flat_far_and_broken_scenes(monkeypatch, name):
    """The parked, far and broken scenes as three problems of one call for every functor (16 registry shapes, Circle, the Polygon
    fallback, the star.obj mesh on a stride of points), with and without the pre-transform, sparse and batched on 3 CTAs: each record
    is the single call's bits."""
    stride = 6 if name == "star_obj_mesh" else 1
    probs = []
    for sname in ("parked", "far", "broken"):
        _, T, co, pts = mko.scene(sname)
        probs.append((T, co, pts[::2 * stride] if sname != "far" else pts[::stride]))
    n_inside = 0
    for pp in PRE:
        for hook in ("sparse", "batched_grid3"):
            ctx = make_ctx(monkeypatch, name, hook, poly_params=pp)
            res = ctx.cost_grad_multi(probs)
            for (T, co, pts), (c, gT, gC, ni) in zip(probs, res):
                assert bits_same(rec_of(c, gT, gC, ni), single_record(ctx, T, co, pts)), (name, pp, hook, len(T))
                n_inside += ni
            ctx.close()
    assert n_inside > 0, name


# ---------------------------------------------------------------------------------------------------------------------
# 4. per-point outputs through svsdf_map_clearance_multi
# ---------------------------------------------------------------------------------------------------------------------
def positions(T, co, ts):
    C = np.asarray(co).reshape(3, len(T), 6).transpose(1, 0, 2)
    return np.array([mko._eval(C, T, t)[:2] for t in ts])


def path_samples(T, co, dt=0.05):
    """Robot positions every dt seconds, at t = D and at every junction (inside the robot: the interior branch)."""
    return positions(T, co, np.r_[np.arange(0.0, float(np.sum(T)), dt), float(np.sum(T)), np.cumsum(T)[:-1]])


def occupancy(xy, res):
    """A 2-D map whose occupied cells contain the points xy: (occ, origin, res)."""
    lo = xy.min(axis=0) - 1.0
    ij = np.floor((xy - lo) / res).astype(np.int64)
    X, Y = (int(v) + 2 for v in ij.max(axis=0))
    occ = np.zeros((X, Y), dtype=bool)
    occ[ij[:, 0], ij[:, 1]] = True
    origin = (float(lo[0]), float(lo[1]))
    return occ, origin, res


@pytest.fixture(scope="module")
def clearance_cases(pinned, oracle_mod):
    """Per robot shape: the trajectories (both ends of parked and endpoints, where the velocity fallback scan runs; the junction and
    broken seams; midstop; the inside of circle_static and circle_spin), a map of the fixture points near the paths and the path
    samples, and clearance_oracle's dense result for each trajectory at d_max = +inf."""
    cases = {}
    for shape, names, res in (("star", ("parked", "endpoints", "junction", "broken", "midstop", "parked"), 0.1),
                              ("Circle", ("circle_static", "circle_spin"), 0.05)):
        trajs = [(pinned[n].T, pinned[n].co) for n in names]
        xy = [path_samples(T, co) for T, co in trajs]
        xy += [pinned[n].pts[np.all(np.abs(pinned[n].pts[:, :2]) < 60.0, axis=1), :2] for n in names]
        occ, origin, res = occupancy(np.concatenate(xy), res)
        want = []
        for T, co in trajs:
            orc = oracle_mod.Oracle(shape, threads=oracle_mod.num_procs())
            orc.set_traj(T, co)
            want.append(clearance_oracle.clearance(orc, occ, origin, res, math.inf))
        cases[shape] = (names, trajs, (occ, origin, res), want)
    return cases


@pytest.mark.parametrize("hook", list(HOOKS))
def test_map_clearance_multi_on_the_edge_trajectories(clearance_cases, monkeypatch, hook):
    """d_max = +inf: every occupied column is evaluated for every trajectory.  Each out[k] is the single map_clearance of trajectory
    k bit for bit (counts, list, sdf, t*, summary) and, in the strict build, clearance_oracle's values."""
    for shape, (names, trajs, (occ, origin, res), want) in clearance_cases.items():
        ctx = make_ctx(monkeypatch, shape, hook)
        tc.set_map(ctx, occ, origin, res)
        got = ctx.map_clearance_multi(trajs, math.inf)
        for name, (T, co), r, w in zip(names, trajs, got, want):
            tcm.same(r, ctx.map_clearance(T, co, math.inf))
            tc.assert_same(r, w)
            assert r.n_evaluated == r.n_occupied == occ.sum() and r.n_colliding > 0, (name, r.n_colliding)
            # the cells under the robot at both ends of the path and at its junctions are inside it
            for p in positions(T, co, np.r_[0.0, float(np.sum(T)), np.cumsum(T)[:-1]]):
                k = int(np.argmin(np.hypot(*(r.xy - p).T)))
                assert r.sdf[k] <= 0.0, (name, p, r.sdf[k])
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. limits and state across calls
# ---------------------------------------------------------------------------------------------------------------------
N_MAX = 65_535  # kMaxMultiProblems: k_finalize_multi's and k_pose_table_multi's grid.y


def small_set(pinned):
    """The distinct one-point problems of the n = 65 535 calls: every tiny_k1 and junction fixture point (N = 1 and 2; tiny_k1's
    interior points included) and four interior points of endpoints (N = 8), so that the interior slots change trajectory."""
    out = [(s.T, s.co, s.pts[k : k + 1]) for s in (pinned["tiny_k1"], pinned["junction"]) for k in range(len(s.pts))]
    e = pinned["endpoints"]
    out += [(e.T, e.co, e.pts[k : k + 1]) for k in np.flatnonzero(e.inside)[:4]]
    assert pinned["tiny_k1"].inside.sum() >= 1
    return out


def records(res):
    return [rec_of(*r) for r in res]


def fresh_multi(monkeypatch, probs):
    ctx = make_ctx(monkeypatch, "star")
    res = records(ctx.cost_grad_multi(probs))
    ctx.close()
    return res


def test_65535_problems_and_65536_refused(pinned, monkeypatch):
    """65 535 one-point problems cycling through the small set: every record is that point's one-problem record (set_points +
    cost_grad on a fresh context).  65 536 problems are refused with SVSDF_ERR_INVALID before any launch."""
    base = small_set(pinned)
    want = []
    for T, co, p in base:
        fresh = make_ctx(monkeypatch, "star")
        want.append(single_record(fresh, T, co, p))
        fresh.close()
    probs = [base[k % len(base)] for k in range(N_MAX)]
    ctx = make_ctx(monkeypatch, "star")
    L = api.lib()
    c_call, c_times, times = L.svsdf_cost_grad_multi, [], []

    def timed(*args):  # the C call alone: host planning, upload, launches, download and the stream synchronise
        t0 = time.perf_counter()
        rc = c_call(*args)
        c_times.append(time.perf_counter() - t0)
        return rc

    monkeypatch.setattr(L, "svsdf_cost_grad_multi", timed)
    for _ in range(2):
        t0 = time.perf_counter()
        res = ctx.cost_grad_multi(probs)
        times.append(time.perf_counter() - t0)
        for k, r in enumerate(res):
            assert bits_same(rec_of(*r), want[k % len(base)]), k
    print(f"\nsvsdf_cost_grad_multi, n = {N_MAX} one-point problems: C call {c_times[0] * 1e3:.1f} ms (first call on the context), "
          f"{c_times[1] * 1e3:.1f} ms (second); with the Python wrapper's packing {times[0] * 1e3:.1f} / {times[1] * 1e3:.1f} ms")
    assert sum(r[3] for r in res) == sum(want[k % len(base)][-1] for k in range(N_MAX)) > 0
    n0 = ctx.kernel_launches()
    with pytest.raises(api.SvsdfError) as e:
        ctx.cost_grad_multi(probs + [base[0]])
    assert "status -1" in str(e.value) and ctx.kernel_launches() == n0
    ctx.close()


def test_sequence_of_calls_on_one_context(pinned, monkeypatch):
    """65 535 -> 3 -> 1 -> 1 439 -> 65 535 problems on one context: the compaction and finalize tickets (zeroed only when their
    buffer grows) must re-arm themselves, the inside flags of a larger earlier call must not leak, and the k_gsip variant follows the
    previous call's interior count (8-warp after more than SMs interior points, 22-warp after fewer).  Every call equals a fresh
    context's bits (a fresh context runs the 8-warp variant)."""
    base = small_set(pinned)
    big = [base[k % len(base)] for k in range(N_MAX)]
    inside = np.flatnonzero(pinned["tiny_k1"].inside)  # the first problems of base are tiny_k1's points
    three = [base[inside[0]], base[len(pinned["tiny_k1"].pts)], base[inside[-1]]]  # interior, junction (none), interior
    one = [base[inside[0]]]
    star = [(s.T, s.co, s.pts[k : k + 1]) for s in pinned.values() if s.shape == "star" for k in range(len(s.pts))]
    seq = [big, three, one, star, big]
    ctx = make_ctx(monkeypatch, "star")
    counts = []
    for probs in seq:
        got = records(ctx.cost_grad_multi(probs))
        want = fresh_multi(monkeypatch, probs)
        assert len(got) == len(want) and all(bits_same(a, b) for a, b in zip(got, want)), len(probs)
        counts.append(int(sum(r[-1] for r in got)))
    ctx.close()
    sms = sm_count()
    wide = [False] + [c <= sms for c in counts[:-1]]  # the variant each call ran: 0 <= previous interior count <= SMs
    print("\ninterior points per call", counts, "22-warp k_gsip_multi", wide)
    assert wide == [False, False, True, True, False], (counts, sms)
