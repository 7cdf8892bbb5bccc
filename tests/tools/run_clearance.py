"""Measures svsdf_map_clearance and runs the benchmark harness the reference declares but stripped (autoBenchMark with getMinSVSDF).

  python tests/tools/run_clearance.py [--reps 5] [--out FILE.jsonl]
  python tests/tools/run_clearance.py --autobench [--problems 256] [--out FILE.jsonl]

Default: band against dense.  The band call (Context.map_clearance) and the dense alternative (svsdf_query, interior branch included, on
the centre of every occupied column, filtered at d_max on the host) run alternately on the same trajectory and map; their outputs must
be identical (the script exits non-zero otherwise).  Scenes: the reference's star scene planned end to end, grid60 plans (the 60 x 60
map of run_plan_batch.py), and a large sparse map (4000 x 4000 cells, 0.1 m, occupancy 0.2 %) around the star-scene plan.
d_max = safety_hor.  Per scene: ms (median; every call ends in a synchronise), n_evaluated / n_occupied, n_within, launches.

--autobench: plan_batch(certify=True) on the grid60 scene for the start / goal pairs of tests/golden/coords.txt
(scenes.make_batch_problems): the share of problems where the front end found a path, where the solver returned status >= 0 and where
the result is collision free against the whole map; the min_sdf distribution; the certification's share of the batch time.

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
from oracle import clearance_oracle  # noqa: E402


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
    return g, cmap, dict(kernel_size=ks, traj_parlength=float(g["traj_parlength"]))


def grid60_scene():
    occ = np.random.default_rng(11).random((60, 60, 1)) < 0.01
    return plan.CloudMap(occ=occ, boundary_min=np.zeros(3), boundary_max=np.array([60.0, 60.0, 1.0]), res=1.0), dict(kernel_size=17)


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def dense(ctx, T, co, occ, origin, res, d_max):
    ij = clearance_oracle.occupied_columns(occ)
    xy = clearance_oracle.centres(ij, origin, res)
    sdf, ts, _, _ = ctx.query(T, co, np.c_[xy, np.zeros(len(xy))], outer_only=False)
    return clearance_oracle.summarise(ij, xy, sdf, ts, d_max, len(ij))


def same(r, d):
    b = lambda a: np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.uint64)  # noqa: E731
    return bool(np.array_equal(r.ij, d["ij"]) and np.array_equal(b(r.xy), b(d["xy"])) and np.array_equal(b(r.sdf), b(d["sdf"]))
                and np.array_equal(b(r.tstar), b(d["tstar"])) and r.argmin == d["argmin"] and r.n_occupied == d["n_occupied"]
                and r.n_colliding == d["n_colliding"] and b(r.min_sdf) == b(d["min_sdf"]))


def set_map(ctx, occ3, origin, res, ks):
    X, Y, Z = occ3.shape
    ctx.set_map3d(plan.pack_map_kernel3d(occ3, ks), X, Y, Z, ks, (origin[0], origin[1], 0.0), res)


def band_vs_dense(reps):
    d_max = scenes.YAML["safety_hor"]
    cases = []
    g, cmap, kw = star_scene()
    ctx = new_ctx()
    p = plan.generate_traj(ctx, cmap, g["start"][:2], g["end"][:2], **kw)
    assert p["ok"], p
    T, co = p["T"], np.asarray(p["coeffs"]).reshape(-1)
    cases.append(("star_scene_plan", ctx, T, co, cmap.occ, cmap.boundary_min[:2], cmap.res, kw["kernel_size"]))
    # large sparse map around the same plan: 400 m x 400 m at 0.1 m
    rng = np.random.default_rng(5)
    big = rng.random((4000, 4000, 1)) < 0.002
    c = np.asarray(p["path"])[:, :2].mean(axis=0)
    cases.append(("large_sparse_4000x4000", ctx, T, co, big, (float(c[0]) - 200.0, float(c[1]) - 200.0), 0.1, kw["kernel_size"]))
    gmap, gkw = grid60_scene()
    gctx = new_ctx()
    sg = scenes.make_batch_problems(16)
    got = plan.plan_batch(gctx, gmap, sg[:, :2], sg[:, 2:], **gkw)
    planned = [r for r in got if "T" in r][:3]
    for k, r in enumerate(planned):
        cases.append((f"grid60_plan{k}", gctx, r["T"], np.asarray(r["coeffs"]).reshape(-1), gmap.occ, (0.0, 0.0), 1.0, gkw["kernel_size"]))
    ok = True
    for name, cx, T, co, occ, origin, res, ks in cases:
        set_map(cx, occ, origin, res, ks)
        cx.map_clearance(T, co, d_max)  # warm-up (buffers grow once)
        dense(cx, T, co, occ, origin, res, d_max)
        n0 = cx.kernel_launches()
        r = cx.map_clearance(T, co, d_max)
        launches = cx.kernel_launches() - n0
        band_ms, dense_ms = [], []
        for _ in range(reps):
            band_ms.append(timed(lambda: cx.map_clearance(T, co, d_max))[0])
            ms, d = timed(lambda: dense(cx, T, co, occ, origin, res, d_max))
            dense_ms.append(ms)
        ident = same(r, d)
        ok &= ident
        rec = dict(scene=name, N=int(len(T)), cells=int(occ.shape[0] * occ.shape[1]), n_occupied=r.n_occupied, n_evaluated=r.n_evaluated,
                   evaluated_share=r.n_evaluated / max(r.n_occupied, 1), n_within=r.n_within, n_colliding=r.n_colliding, min_sdf=r.min_sdf,
                   launches=int(launches), band_ms=float(np.median(band_ms)), dense_ms=float(np.median(dense_ms)), identical=ident)
        yield rec
    ctx.close()
    gctx.close()
    if not ok:
        raise SystemExit("band and dense results differ")


def autobench(n):
    gmap, kw = grid60_scene()
    sg = scenes.make_batch_problems(n)
    ctx = new_ctx()
    stats = {}
    t0 = time.perf_counter()
    out = plan.plan_batch(ctx, gmap, sg[:, :2], sg[:, 2:], certify=True, stats=stats, **kw)
    wall = time.perf_counter() - t0
    ctx.close()
    found = [r for r in out if "path" in r]
    solved = [r for r in out if "status" in r and r["status"] >= 0]
    cert = [r["clearance"] for r in out if "clearance" in r]
    free = [c for c in cert if c["collision_free"]]
    solved_free = [r for r in solved if r["clearance"]["collision_free"]]
    m = np.array([c["min_sdf"] for c in cert])
    fin = m[np.isfinite(m)]
    q = lambda v: float(np.percentile(fin, v))  # noqa: E731
    return dict(mode="autobench", scene="grid60", problems=n, front_end_path=len(found) / n, solver_ok=len(solved) / n,
                collision_free=len(free) / n, solver_ok_and_collision_free=len(solved_free) / n, certified=len(cert),
                colliding_plans=len(cert) - len(free), min_sdf_inf=int(np.sum(~np.isfinite(m))),
                min_sdf_percentiles={"p0": q(0), "p5": q(5), "p25": q(25), "p50": q(50), "p75": q(75), "p100": q(100)} if fin.size else None,
                n_within_mean=float(np.mean([c["n_within"] for c in cert])) if cert else None,
                batch_s=wall, certify_s=stats.get("certify_s", 0.0), certify_share=stats.get("certify_s", 0.0) / wall,
                stages_s={k: stats[k] for k in ("front_s", "points_s", "mid_s", "back_s")})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--autobench", action="store_true")
    ap.add_argument("--problems", type=int, default=256)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    info = gpu_info()
    recs = [autobench(a.problems)] if a.autobench else band_vs_dense(a.reps)
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
