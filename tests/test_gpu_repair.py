"""GPU (-m gpu): collision repair.  generate_traj(repair=R) against the same loop written out with public calls (map_clearance,
plan.new_cells, set_points(points ++ added), optimize from the previous x), bit for bit; repair=0 against today's result, key for key;
plan_batch(repair=3) against generate_traj(repair=3) per problem, bit for bit, on the reference's star scene and on the grid60 scene with
the first 32 pairs of tests/golden/coords.txt, and on grid60 with kernel size 3, where first certificates do list cells outside the query
set; certify=True in plan_batch through svsdf_map_clearance_multi; "closed" means the last certificate has no new cell."""
import os

import numpy as np
import pytest

import test_gpu_clearance as tc
from implicit_svsdf_planner_b200 import api, plan, scenes

pytestmark = pytest.mark.gpu
same_value = tc.same_value
PARAMS = api.default_lbfgs_params(mem_size=16, past=3, delta=1e-6, g_epsilon=0.0, max_iterations=0, min_step=1e-32)
TRAJ_KEYS = ("T", "coeffs", "x", "final_cost", "status", "ok", "iterations", "evaluations")


def grid60_scene():
    occ = np.random.default_rng(11).random((60, 60, 1)) < 0.01  # the map of tests/tools/run_plan_batch.py and run_clearance.py
    return plan.CloudMap(occ=occ, boundary_min=np.zeros(3), boundary_max=np.array([60.0, 60.0, 1.0]), res=1.0), dict(kernel_size=17)


@pytest.fixture(scope="module")
def star():
    """The reference's star scene: its own start / goal, then 5 seeded pairs of free cells."""
    g = np.load(os.path.join(tc.GOLD, "map_star_pcd.npz"))
    res, ks = float(g["occupancy_resolution"]), int(g["kernel_size"])
    cmap = plan.gridmap3d_from_cloud(g["points"], res, int(g["sta_threshold"]))
    free = np.argwhere(~cmap.occ.any(axis=2))
    pick = free[np.random.default_rng(7).choice(len(free), size=(5, 2), replace=False)]
    xy = cmap.boundary_min[:2] + (pick + 0.5) * cmap.res
    kw = dict(kernel_size=ks, traj_parlength=float(g["traj_parlength"]))
    return cmap, kw, np.r_[[g["start"][:2]], xy[:, 0]], np.r_[[g["end"][:2]], xy[:, 1]]


@pytest.fixture(scope="module")
def grid60():
    cmap, kw = grid60_scene()
    sg = scenes.make_batch_problems(32)
    return cmap, kw, sg[:, :2], sg[:, 2:]


@pytest.fixture(scope="module")
def grid60_ks3(grid60):
    """grid60 with kernel size 3: waypoint boxes of half-width res (one cell on each side), far smaller than the star robot, so the
    certificate lists occupied cells near the path that no box holds.  (On the star scene's six pairs and the first 32 grid60 pairs with
    kernel size 17 the boxes hold every cell within safety_hor of the first plans: no first certificate there lists a new cell.)"""
    cmap, kw, st, go = grid60
    return cmap, dict(kw, kernel_size=3), st, go


def written_out(ctx, cmap, s, e, kw, R):
    """generate_traj(repair=R) restated: today's plan, then the rounds with public calls only."""
    p = plan.generate_traj(ctx, cmap, s, e, **kw)
    if "T" not in p:
        return p, None
    pts = ctx.get_points()
    path = p["path"]
    init_s, final_s = np.zeros((3, 3)), np.zeros((3, 3))
    init_s[:, 0], final_s[:, 0] = path[0], path[-1]
    x, T, b, added, mins = p["x"], p["T"], p["coeffs"], [], []
    while True:
        cl = ctx.map_clearance(T, np.asarray(b).reshape(-1), ctx.safety_hor)
        mins.append(cl.min_sdf)
        new = plan.new_cells(cl.xy, pts)
        if len(new) == 0 or len(added) == R:
            break
        added.append(new)
        pts = np.r_[pts, new]
        ctx.set_points(pts)
        rc, x, T, b, st = ctx.optimize(init_s, final_s, x, p["N"], PARAMS)
        p.update(ok=rc >= 0, status=int(rc), final_cost=float(st["final_cost"]), iterations=int(st["iterations"]),
                 evaluations=int(st["evaluations"]), T=T, coeffs=b, x=x)
    return p, dict(cl=cl, added=added, mins=mins, closed=len(new) == 0, points=pts)


def check_single(ctx, cmap, s, e, kw, R=3):
    p, w = written_out(ctx, cmap, s, e, kw, R)
    r = plan.generate_traj(ctx, cmap, s, e, repair=R, **kw)
    if w is None:
        assert "repair" not in r
        return r, 0
    for k in TRAJ_KEYS:
        assert same_value(r[k], p[k]), k
    rp = r["repair"]
    assert rp["rounds"] == len(w["added"]) and rp["added_per_round"] == [len(a) for a in w["added"]]
    assert same_value(rp["added"], np.concatenate(w["added"]) if w["added"] else np.empty((0, 2)))
    assert [tc.bits(v) for v in rp["min_sdf_per_round"]] == [tc.bits(v) for v in w["mins"]]
    assert rp["stopped"] == ("closed" if w["closed"] else "limit")
    assert same_value(r["clearance"], plan.certificate_of(w["cl"]))
    assert np.array_equal(tc.bits(ctx.get_points()), tc.bits(w["points"]))  # the resident set is the last query set
    if rp["stopped"] == "closed":  # the last certificate lists no cell outside the last query set
        assert len(plan.new_cells(ctx.map_clearance(r["T"], np.asarray(r["coeffs"]).reshape(-1), ctx.safety_hor).xy, w["points"])) == 0
    return r, rp["added_per_round"][0] if rp["rounds"] else 0


def test_repair_zero_is_today(star):
    cmap, kw, st, go = star
    ctx = tc.new_ctx()
    for certify in (False, True):
        a = plan.generate_traj(ctx, cmap, st[0], go[0], certify=certify, **kw)
        b = plan.generate_traj(ctx, cmap, st[0], go[0], certify=certify, repair=0, **kw)
        assert a.keys() == b.keys() and "repair" not in b
        for k in a:
            if k != "seconds":
                assert same_value(a[k], b[k]), k
    ctx.close()


@pytest.mark.parametrize("scene", ["star", "grid60", "grid60_ks3"])
def test_repair_is_its_definition_and_batch_equals_single(scene, request):
    cmap, kw, st, go = request.getfixturevalue(scene)
    ctx = tc.new_ctx()
    stats = {}
    batch = plan.plan_batch(tc.new_ctx(), cmap, st, go, repair=3, stats=stats, **kw)
    assert stats["repair_s"] >= 0.0 and stats["certify_s"] > 0.0 and 0 <= stats["repair_rounds"] <= 3
    gained = 0
    for s, e, b in zip(st, go, batch):
        r, first = check_single(ctx, cmap, s, e, kw)
        gained += first > 0
        assert ("repair" in b) == ("repair" in r) == ("T" in r)
        if "repair" in r:
            for k in TRAJ_KEYS + ("clearance", "repair", "n_points", "N"):
                assert same_value(b[k], r[k]), k
    if scene == "grid60_ks3":  # not vacuous: first certificates listed cells that were not query points
        assert gained > 0
    assert stats["repair_rounds"] == max([b["repair"]["rounds"] for b in batch if "repair" in b] + [0])
    ctx.close()


def test_plan_batch_certify_unchanged_by_the_multi_entry(grid60):
    """certify=True alone: the clearance of every problem equals generate_traj(certify=True)'s, and no `repair` key appears."""
    cmap, kw, st, go = grid60
    ctx = tc.new_ctx()
    batch = plan.plan_batch(tc.new_ctx(), cmap, st[:8], go[:8], certify=True, **kw)
    for s, e, b in zip(st[:8], go[:8], batch):
        alone = plan.generate_traj(ctx, cmap, s, e, certify=True, **kw)
        assert "repair" not in b and ("clearance" in b) == ("clearance" in alone)
        if "clearance" in b:
            assert same_value(b["clearance"], alone["clearance"])
    ctx.close()
