"""GPU (-m gpu): plan.plan_batch on the reference's star scene (tests/golden/map_star_pcd.npz) — every problem's result is the one
plan.generate_traj gives it alone, bit for bit, and every failure says why."""
import os

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, plan, scenes

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.uint64)


@pytest.fixture(scope="module")
def scene():
    g = np.load(os.path.join(HERE, "golden", "map_star_pcd.npz"))
    res, ks = float(g["occupancy_resolution"]), int(g["kernel_size"])
    cmap = plan.gridmap3d_from_cloud(g["points"], res, int(g["sta_threshold"]))
    free = np.argwhere(~cmap.occ.any(axis=2))
    rng = np.random.default_rng(7)
    pick = free[rng.choice(len(free), size=(56, 2), replace=False)]
    xy = cmap.boundary_min[:2] + (pick + 0.5) * res
    starts, goals = [g["start"][:2]] + list(xy[:, 0]), [g["end"][:2]] + list(xy[:, 1])
    starts.append(np.array([-1e3, -1e3]))  # outside the map
    goals.append(g["end"][:2])
    occ = np.argwhere(cmap.occ.any(axis=2))
    if len(occ):  # a goal on an occupied cell: no path
        starts.append(g["start"][:2])
        goals.append(cmap.boundary_min[:2] + (occ[len(occ) // 2] + 0.5) * res)
    return g, cmap, res, ks, np.array(starts), np.array(goals)


def ctx_new():
    return api.Context("star", weight_p=scenes.YAML["weight_p"], safety_hor=scenes.YAML["safety_hor"], rho=scenes.YAML["rho"])


@pytest.mark.parametrize("max_path,max_in_flight", [(4096, 0), (40, 3)])
def test_plan_batch_equals_generate_traj(scene, max_path, max_in_flight):
    g, cmap, res, ks, starts, goals = scene
    kw = dict(kernel_size=ks, traj_parlength=float(g["traj_parlength"]), max_path=max_path)
    ctx = ctx_new()
    got = plan.plan_batch(ctx, cmap, starts, goals, max_in_flight=max_in_flight, **kw)
    _, _, dev_status, _ = ctx.front_astar_device(starts, goals, max_path)
    dev_paths_long = ctx.front_astar_device(starts, goals, 4096)[0]
    ok = 0
    reasons = set()
    for q in range(len(starts)):
        ref_ctx = ctx_new()
        r = plan.generate_traj(ref_ctx, cmap, starts[q], goals[q], **kw)
        b = got[q]
        assert b["ok"] == r["ok"], (q, b.get("reason"), r.get("reason"))
        if not r["ok"]:
            reasons.add(b["reason"])
            if "mid end" in r["reason"]:
                assert b["reason"] == r["reason"]
            else:  # generate_traj's lock-step search says only that there is no path; the device search says why
                assert r["reason"] == "front end found no path"
                st = dev_status[q]
                want = {0: "start or goal outside the map", 1: "front end found no path", 2: "front end found no path",
                        3: "front end reached max_expansions", 4: "path longer than max_path"}[st]
                assert b["reason"] == want and b["astar_status"] == st, (q, b, st)
                inside = all(cmap.boundary_min[a] <= v[a] <= cmap.boundary_min[a] + cmap.occ.shape[a] * res
                             for v in (starts[q], goals[q]) for a in (0, 1))
                assert (st == 0) == (not inside), q
                if st == 4:
                    full = dev_paths_long[q]  # the same search without the length cap is longer than max_path
                    assert full is not None and len(full) > max_path, q
            ref_ctx.close()
            continue
        ok += 1
        for key in ("path", "waypoints", "x", "T", "coeffs"):
            assert np.array_equal(bits(b[key]), bits(r[key])), (q, key)
        for key in ("N", "n_points", "status", "iterations", "evaluations", "expansions"):
            assert b[key] == r[key], (q, key, b[key], r[key])
        for key in ("final_cost", "cost_at_warm_start"):
            assert bits(b[key]) == bits(r[key]), (q, key)
        assert b["mid"]["status"] == r["mid"]["status"] and b["mid"]["iterations"] == r["mid"]["iterations"]
        assert bits(b["mid"]["cost"]) == bits(r["mid"]["cost"]) and np.array_equal(bits(b["mid"]["T"]), bits(r["mid"]["T"]))
        assert np.array_equal(bits(b["points"]), bits(ref_ctx.get_points())), q
        ref_ctx.close()
    assert ok >= 3
    assert "start or goal outside the map" in reasons
    if max_path == 40:
        assert "path longer than max_path" in reasons
    ctx.close()


def test_a_failing_mid_end_fails_its_problem_only(scene):
    """generate_traj raises when the mid end refuses its input; plan_batch marks each such problem failed instead of aborting the batch."""
    g, cmap, res, ks, starts, goals = scene
    kw = dict(kernel_size=ks, traj_parlength=float(g["traj_parlength"]))
    bad = api.mid_default_config(integralIntervs=0)  # refused by svsdf_mid_get_ori_traj
    ctx = ctx_new()
    got = plan.plan_batch(ctx, cmap, starts[:6], goals[:6], mid_cfg=bad, **kw)
    found = [b for b in got if b.get("reason") != "front end found no path" and "outside" not in b.get("reason", "")
             and "max_path" not in b.get("reason", "")]
    assert found and all(not b["ok"] and b["reason"].startswith("mid end failed") for b in found)
    with pytest.raises(api.SvsdfError):
        plan.generate_traj(ctx_new(), cmap, starts[0], goals[0], mid_cfg=bad, **kw)
    ctx.close()
