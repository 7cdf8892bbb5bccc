"""Measures svsdf_swept_contour_multi against a loop of svsdf_swept_contour calls on the final trajectories of plan_batch.

  python tests/tools/run_swept_multi.py [--sizes 256,1024] [--hs 0.2,0.05] [--reps 3] [--out FILE.jsonl]

Scenes: the reference's star scene (tests/golden/map_star_pcd.npz, seeded start / goal pairs on free cells, drawn as run_plan_batch.py draws
them) and grid60 (the 60 x 60 map of run_plan_batch.py with the pairs of tests/golden/coords.txt, scenes.make_batch_problems).  For each
scene and size, plan_batch runs once; the outlines of every problem that went through the back end are then made at iso = safety_hor,
strict build, for each h, by a loop of single calls and by one multi call, alternately, reps times (every call ends in a synchronise);
the median of each is printed.  The two must give identical outputs (the script exits non-zero otherwise).  Every line also holds the
GPU's name, power limit and max SM clock, read in the same process."""
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
    return api.Context("star", weight_p=scenes.YAML["weight_p"], safety_hor=scenes.YAML["safety_hor"], rho=scenes.YAML["rho"], strict_fp=True)


def star_scene(n):
    g = np.load(os.path.join(ROOT, "tests", "golden", "map_star_pcd.npz"))
    res, ks = float(g["occupancy_resolution"]), int(g["kernel_size"])
    cmap = plan.gridmap3d_from_cloud(g["points"], res, int(g["sta_threshold"]))
    free = np.argwhere(~cmap.occ.any(axis=2))
    pick = free[np.random.default_rng(1000 + n).integers(0, len(free), size=(n, 2))]
    xy = cmap.boundary_min[:2] + (pick + 0.5) * cmap.res
    return cmap, dict(kernel_size=ks, traj_parlength=float(g["traj_parlength"])), xy[:, 0].copy(), xy[:, 1].copy()


def grid60_scene(n):
    occ = np.random.default_rng(11).random((60, 60, 1)) < 0.01
    cmap = plan.CloudMap(occ=occ, boundary_min=np.zeros(3), boundary_max=np.array([60.0, 60.0, 1.0]), res=1.0)
    sg = scenes.make_batch_problems(n)
    return cmap, dict(kernel_size=17), sg[:, :2], sg[:, 2:]


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.uint64)


def same(a, b):
    return bool((a.i0, a.j0, a.nx, a.ny, a.clipped, a.n_evaluated) == (b.i0, b.j0, b.nx, b.ny, b.clipped, b.n_evaluated)
                and np.array_equal(bits(a.vertices), bits(b.vertices)) and np.array_equal(a.segments, b.segments)
                and np.array_equal(a.triangles, b.triangles))


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="256,1024")
    ap.add_argument("--hs", default="0.2,0.05")
    ap.add_argument("--scenes", default="star,grid60")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    info = gpu_info()
    iso = scenes.YAML["safety_hor"]
    ok = True
    lines = []
    for scene in a.scenes.split(","):
        for n in (int(s) for s in a.sizes.split(",")):
            cmap, kw, st, go = (star_scene if scene == "star" else grid60_scene)(n)
            ctx = new_ctx()
            res = plan.plan_batch(ctx, cmap, st, go, **kw)
            trajs = [(r["T"], np.asarray(r["coeffs"]).reshape(-1)) for r in res if "T" in r]
            for h in (float(v) for v in a.hs.split(",")):
                loop = lambda: [ctx.swept_contour(T, co, h, iso) for T, co in trajs]  # noqa: E731
                multi = lambda: ctx.swept_contour_multi(trajs, h, iso)  # noqa: E731
                loop()
                multi()  # warm-up: buffers grow once
                n0 = ctx.kernel_launches()
                multi()
                launches_multi = ctx.kernel_launches() - n0
                loop_ms, multi_ms = [], []
                for _ in range(a.reps):
                    ms, lo = timed(loop)
                    loop_ms.append(ms)
                    ms, mu = timed(multi)
                    multi_ms.append(ms)
                ident = len(lo) == len(mu) and all(same(x, y) for x, y in zip(lo, mu))
                ok &= ident
                rec = dict(scene=scene, pairs=n, plans=len(trajs), h=h, iso=iso, corners=int(sum(m.nx * m.ny for m in mu)),
                           evaluated=int(sum(m.n_evaluated for m in mu)), launches_multi=int(launches_multi),
                           loop_ms=float(np.median(loop_ms)), multi_ms=float(np.median(multi_ms)),
                           speedup=float(np.median(loop_ms) / np.median(multi_ms)), identical=ident, **info)
                print(json.dumps(rec), flush=True)
                lines.append(rec)
            ctx.close()
    if a.out:
        with open(a.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
