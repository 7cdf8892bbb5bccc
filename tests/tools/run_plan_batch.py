"""Batch planning measurement: n start / goal problems on one map, solved three ways in the same process.

  loop     plan.generate_traj per problem, one context (lock-step A* per problem, one back end at a time)
  pool     the plan_batch chain (device A* for all searches, extraction, mid end) with the back end on a pool of 3 contexts on the
           GPU: three host threads, each optimising one problem at a time with svsdf_optimize (the pool of svsdf_optimize_batch)
  batch    plan.plan_batch: the same front and mid end, then ONE lock-step back end (svsdf_optimize_lockstep, its L-BFGS machines
           advanced round by round on the host; svsdf_optimize_device from plan.DEVICE_BACK_END_MIN_PROBLEMS problems)

Scenes: the reference's star scene (tests/golden/map_star_pcd.npz) and a 60 x 60 map at resolution 1.0 (seeded obstacles, density
0.01, one z layer); seeded start / goal pairs on free cells.  Every problem's result must be identical in the three ways (path, N,
x, T, coefficients, status, iterations, evaluations, final cost) or the script exits non-zero.  Prints one JSON line per (scene, n):
wall seconds per batch of each way, the batch way's stage split, rounds and launches per round, the back end's share of the time,
and the GPU's name, power limit and max SM clock (read with nvidia-smi queries).

    python tests/tools/run_plan_batch.py [--sizes 256,1024] [--loop-max 1024] [--scenes star,grid60]
"""
import argparse
import concurrent.futures as cf
import json
import os
import queue
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from implicit_svsdf_planner_b200 import api, plan, scenes  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = (v.strip() for v in r.stdout.splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def new_ctx():
    return api.Context("star", weight_p=scenes.YAML["weight_p"], safety_hor=scenes.YAML["safety_hor"], rho=scenes.YAML["rho"])


def star_scene():
    g = np.load(os.path.join(ROOT, "tests", "golden", "map_star_pcd.npz"))
    res, ks = float(g["occupancy_resolution"]), int(g["kernel_size"])
    return plan.gridmap3d_from_cloud(g["points"], res, int(g["sta_threshold"])), dict(kernel_size=ks, traj_parlength=float(g["traj_parlength"]))


def grid60_scene():
    occ = np.random.default_rng(11).random((60, 60, 1)) < 0.01
    return plan.CloudMap(occ=occ, boundary_min=np.zeros(3), boundary_max=np.array([60.0, 60.0, 1.0]), res=1.0), dict(kernel_size=17)


def pairs(cmap, n, seed):
    free = np.argwhere(~cmap.occ.any(axis=2))
    rng = np.random.default_rng(seed)
    pick = free[rng.integers(0, len(free), size=(n, 2))]
    xy = cmap.boundary_min[:2] + (pick + 0.5) * cmap.res
    return xy[:, 0].copy(), xy[:, 1].copy()


KEYS = ("x", "T", "coeffs")


def same(a, b):
    if a["ok"] != b["ok"]:
        return False
    if not a["ok"]:
        return True
    if any(not np.array_equal(np.asarray(a[k]).view(np.uint64), np.asarray(b[k]).view(np.uint64)) for k in KEYS + ("path",)):
        return False
    return all(a[k] == b[k] for k in ("N", "status", "iterations", "evaluations")) and \
        np.float64(a["final_cost"]).view(np.uint64) == np.float64(b["final_cost"]).view(np.uint64)


def run_loop(cmap, kw, st, go):
    ctx = new_ctx()
    t0 = time.perf_counter()
    out = [plan.generate_traj(ctx, cmap, st[q], go[q], **kw) for q in range(len(st))]
    wall = time.perf_counter() - t0
    ctx.close()
    back = sum(r.get("seconds", 0.0) for r in out)
    return out, wall, back


PARAMS = dict(mem_size=16, past=3, delta=1e-6, g_epsilon=0.0, min_step=1e-32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="256,1024")
    ap.add_argument("--loop-max", type=int, default=1 << 30, help="run the generate_traj loop only for n up to this")
    ap.add_argument("--scenes", default="star,grid60")
    a = ap.parse_args()
    info = gpu_info()
    params = api.default_lbfgs_params(max_iterations=0, **PARAMS)
    ok = True
    for name in a.scenes.split(","):
        cmap, kw = star_scene() if name == "star" else grid60_scene()
        for n in (int(s) for s in a.sizes.split(",")):
            st, go = pairs(cmap, n, 1000 + n)
            ctx = new_ctx()
            stats = {}
            t0 = time.perf_counter()
            batch = plan.plan_batch(ctx, cmap, st, go, stats=stats, **kw)
            wall_batch = time.perf_counter() - t0
            ctx.close()
            rec = {"scene": name, "n": n, "ok": int(sum(r["ok"] for r in batch)),
                   "batch_s": wall_batch, "batch_stages_s": {k: stats[k] for k in ("front_s", "points_s", "mid_s", "back_s")},
                   "batch_back_share": stats["back_s"] / wall_batch, "rounds": stats["rounds"],
                   "launches_per_round": stats["back_launches"] / max(stats["rounds"], 1), **info}
            pool, wall_pool, back_pool = run_pool_from(cmap, kw, st, go, params)
            rec.update(pool_s=wall_pool, pool_back_share=back_pool / wall_pool,
                       pool_identical=all(same(x, y) for x, y in zip(batch, pool)))
            ok &= rec["pool_identical"]
            if n <= a.loop_max:
                loop, wall_loop, back_loop = run_loop(cmap, kw, st, go)
                rec.update(loop_s=wall_loop, loop_back_share=back_loop / wall_loop, loop_identical=all(same(x, y) for x, y in zip(batch, loop)))
                ok &= rec["loop_identical"]
            print(json.dumps(rec), flush=True)
    sys.exit(0 if ok else 1)


def run_pool_from(cmap, kw, st, go, params):
    """The pool arm: plan_batch's front and mid end (timed), then the back ends on 3 contexts (3 host threads)."""
    ctx = new_ctx()
    stats = {}
    t0 = time.perf_counter()
    inputs = plan.plan_batch(ctx, cmap, st, go, stats=stats, back_end=False, **kw)
    t_front = time.perf_counter() - t0 - stats["back_s"]
    ctx.close()
    pool = [new_ctx() for _ in range(3)]
    free = queue.Queue()
    for c in pool:
        free.put(c)

    def one(r):
        c = free.get()
        try:
            rc, x, T, b, s = c_optimize(c, r, params)
            return dict(r, ok=rc >= 0, status=int(rc), x=x, T=T, coeffs=b, final_cost=s["final_cost"], iterations=s["iterations"],
                        evaluations=s["evaluations"])
        finally:
            free.put(c)

    todo = [r for r in inputs if "x0" in r]
    t1 = time.perf_counter()
    with cf.ThreadPoolExecutor(max_workers=3) as ex:
        done = dict(zip([id(r) for r in todo], ex.map(one, todo)))
    t_back = time.perf_counter() - t1
    for c in pool:
        c.close()
    return [done.get(id(r), r) for r in inputs], t_front + t_back, t_back


def c_optimize(ctx, r, params):
    ctx.set_points(r["points"])
    return ctx.optimize(r["init_s"], r["final_s"], r["x0"], r["N"], params)


if __name__ == "__main__":
    main()
