"""Measures svsdf_map_clearance_multi and the repair rounds of plan_batch.

  python tests/tools/run_repair.py [--sizes 256,1024] [--reps 3] [--out FILE.jsonl]
  python tests/tools/run_repair.py --autobench [--problems 256] [--repair 3] [--out FILE.jsonl]

Default: the per-problem loop of Context.map_clearance against one Context.map_clearance_multi on the same trajectories (the plans of
plan_batch on the grid60 scene, tests/golden/coords.txt pairs, and on the reference's star scene, seeded free-cell pairs), d_max =
safety_hor.  Both run alternately; their outputs must be identical (the script exits non-zero otherwise).  Per scene and n: wall ms
(median; both calls end in a stream synchronise), kernel launches, band cells.

--autobench: plan_batch(repair=R) on the grid60 scene for the first n coords pairs: plans whose certificate lists cells outside the query
set, and colliding plans, before the first repair round and after the last; the rounds; the repair's share of the batch time.

Every line also holds the GPU's name, power limit and max SM clock, read in the same process."""
import argparse
import json
import os
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
    cmap = plan.gridmap3d_from_cloud(g["points"], res, int(g["sta_threshold"]))
    return cmap, dict(kernel_size=ks, traj_parlength=float(g["traj_parlength"]))


def grid60_scene():
    occ = np.random.default_rng(11).random((60, 60, 1)) < 0.01
    return plan.CloudMap(occ=occ, boundary_min=np.zeros(3), boundary_max=np.array([60.0, 60.0, 1.0]), res=1.0), dict(kernel_size=17)


def pairs(name, cmap, n):
    if name == "grid60":
        sg = scenes.make_batch_problems(n)
        return sg[:, :2], sg[:, 2:]
    free = np.argwhere(~cmap.occ.any(axis=2))
    pick = free[np.random.default_rng(1000 + n).integers(0, len(free), size=(n, 2))]
    xy = cmap.boundary_min[:2] + (pick + 0.5) * cmap.res
    return xy[:, 0].copy(), xy[:, 1].copy()


def identical(a, b):
    u = lambda v: np.ascontiguousarray(np.asarray(v, dtype=np.float64)).view(np.uint64)  # noqa: E731
    return bool(np.array_equal(a.ij, b.ij) and np.array_equal(u(a.xy), u(b.xy)) and np.array_equal(u(a.sdf), u(b.sdf))
                and np.array_equal(u(a.tstar), u(b.tstar)) and (a.n_occupied, a.n_evaluated, a.n_within, a.n_colliding, a.argmin)
                == (b.n_occupied, b.n_evaluated, b.n_within, b.n_colliding, b.argmin) and u(a.min_sdf) == u(b.min_sdf))


def loop_vs_multi(sizes, reps):
    d_max = scenes.YAML["safety_hor"]
    ok = True
    for name in ("grid60", "star"):
        cmap, kw = grid60_scene() if name == "grid60" else star_scene()
        st, go = pairs(name, cmap, max(sizes))
        ctx = new_ctx()
        got = plan.plan_batch(ctx, cmap, st, go, **kw)  # sets the context's map
        trajs = [(r["T"], np.asarray(r["coeffs"]).reshape(-1)) for r in got if "T" in r]
        for n in sizes:
            tr = trajs[:n]
            multi = ctx.map_clearance_multi(tr, d_max)  # warm-up: buffers grow once
            loop = [ctx.map_clearance(T, co, d_max) for T, co in tr]
            n0 = ctx.kernel_launches()
            ctx.map_clearance_multi(tr, d_max)
            l_multi = ctx.kernel_launches() - n0
            n0 = ctx.kernel_launches()
            [ctx.map_clearance(T, co, d_max) for T, co in tr]
            l_loop = ctx.kernel_launches() - n0
            t_loop, t_multi = [], []
            for _ in range(reps):
                t0 = time.perf_counter()
                loop = [ctx.map_clearance(T, co, d_max) for T, co in tr]
                t1 = time.perf_counter()
                multi = ctx.map_clearance_multi(tr, d_max)
                t2 = time.perf_counter()
                t_loop.append((t1 - t0) * 1e3)
                t_multi.append((t2 - t1) * 1e3)
            same = all(identical(a, b) for a, b in zip(loop, multi))
            ok &= same
            yield dict(mode="loop_vs_multi", scene=name, n=len(tr), loop_ms=float(np.median(t_loop)), multi_ms=float(np.median(t_multi)),
                       speedup=float(np.median(t_loop) / np.median(t_multi)), loop_launches=int(l_loop), multi_launches=int(l_multi),
                       band_cells=int(sum(c.n_evaluated for c in multi)), n_occupied=int(multi[0].n_occupied) if multi else 0,
                       identical=same)
        ctx.close()
    if not ok:
        raise SystemExit("map_clearance and map_clearance_multi differ")


def autobench(n, R, ks):
    cmap, kw = grid60_scene()
    kw["kernel_size"] = ks
    st, go = pairs("grid60", cmap, n)
    ctx = new_ctx()
    stats = {}
    t0 = time.perf_counter()
    out = plan.plan_batch(ctx, cmap, st, go, repair=R, stats=stats, **kw)
    wall = time.perf_counter() - t0
    ctx.close()
    rep = [r for r in out if "repair" in r]
    rounds = [r["repair"]["rounds"] for r in rep]
    return dict(mode="autobench", scene="grid60", kernel_size=ks, problems=n, repair=R, certified=len(rep),
                new_cells_before=sum(k > 0 for k in rounds), new_cells_after=sum(r["repair"]["stopped"] == "limit" for r in rep),
                colliding_before=sum(r["repair"]["min_sdf_per_round"][0] <= 0.0 for r in rep),
                colliding_after=sum(not r["clearance"]["collision_free"] for r in rep),
                solver_ok_after=sum(r["ok"] for r in rep), rounds_hist={str(k): rounds.count(k) for k in sorted(set(rounds))},
                added_cells=int(sum(len(r["repair"]["added"]) for r in rep)), repair_rounds=stats.get("repair_rounds", 0),
                batch_s=wall, certify_s=stats["certify_s"], repair_s=stats.get("repair_s", 0.0), repair_share=stats.get("repair_s", 0.0) / wall,
                stages_s={k: stats[k] for k in ("front_s", "points_s", "mid_s", "back_s")})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="256,1024")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--autobench", action="store_true")
    ap.add_argument("--problems", type=int, default=256)
    ap.add_argument("--repair", type=int, default=3)
    ap.add_argument("--kernel-size", type=int, default=17, help="--autobench: the map kernel size (17: the grid60 scene's)")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    info = gpu_info()
    recs = [autobench(a.problems, a.repair, a.kernel_size)] if a.autobench else loop_vs_multi([int(s) for s in a.sizes.split(",")], a.reps)
    lines = []
    for rec in recs:
        rec.update(info)
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    if a.out:
        with open(a.out, "w") as fh:
            for rec in lines:
                fh.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
