"""Measures svsdf_swept_contour (narrow band) against the dense alternative (svsdf_query(outer_only) on every corner of the same grid,
then the same contouring on the CPU) and checks that both give the same mesh.  One JSON line per (scene, h), then one line with the card.

  python tests/tools/run_swept.py [--reps 5] [--dense-max 6000000] [--out FILE.jsonl]

Scenes: the reference's star scene planned end to end (plan.generate_traj), the config-2 trajectory (star, N = 8) and the config-4m
trajectory (sdHorseshoe scene, N = 16) through the reference's star.obj mesh functor.  h in {0.05, 0.02, 0.01}, iso = safety_hor.
Per call: ms (median over repetitions; band and dense alternate, every call ends in a synchronise), corners in the box, corners
evaluated, executed lane evaluations (svsdf_executed_evals), kernel launches, V / S / F."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from implicit_svsdf_planner_b200 import api, plan, scenes  # noqa: E402
from oracle import swept_py  # noqa: E402


def star_plan():
    g = np.load(os.path.join(ROOT, "tests", "golden", "map_star_pcd.npz"))
    res, ks = float(g["occupancy_resolution"]), int(g["kernel_size"])
    cmap = plan.gridmap3d_from_cloud(g["points"], res, int(g["sta_threshold"]))
    ctx = api.Context("star", weight_p=scenes.YAML["weight_p"], safety_hor=scenes.YAML["safety_hor"], rho=scenes.YAML["rho"])
    p = plan.generate_traj(ctx, cmap, g["start"][:2], g["end"][:2], kernel_size=ks, traj_parlength=float(g["traj_parlength"]))
    assert p["ok"], p
    return ctx, p["T"], np.asarray(p["coeffs"]).reshape(-1)


def config(shape, N, mesh=None, scene_shape=None):
    sc = scenes.make_scene(scene_shape or shape, N, 10)
    ctx = api.Context(shape, weight_p=sc.weight_p, safety_hor=sc.safety_hor, rho=sc.rho, mesh=mesh)
    return ctx, sc.T, sc.coeffs_colmajor()


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def dense_contour(ctx, T, co, r, iso):
    x, y = r.corners()
    X, Y = np.meshgrid(x, y)
    f = ctx.query(T, co, np.c_[X.reshape(-1), Y.reshape(-1), np.zeros(X.size)], outer_only=True)[0].reshape(r.ny, r.nx)
    return swept_py.swept_contour(f, r.i0, r.j0, r.h, iso)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--dense-max", type=int, default=6_000_000)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    g = np.load(os.path.join(ROOT, "tests", "golden", "fwn_ref.npz"))
    scenes_ = [("star_scene_plan", star_plan), ("config2", lambda: config("star", 8)),
               ("config4m", lambda: config("star_obj_mesh_sdf", 16, mesh=(g["star_V"], g["star_F"]), scene_shape="sdHorseshoe"))]
    iso = scenes.YAML["safety_hor"]
    lines = []
    for name, make in scenes_:
        ctx, T, co = make()
        for h in (0.05, 0.02, 0.01):
            ctx.swept_contour(T, co, h, iso)  # warm-up (buffers grow once)
            ctx.executed_evals(True)
            n0 = ctx.kernel_launches()
            r = ctx.swept_contour(T, co, h, iso)
            launches = ctx.kernel_launches() - n0
            evals = ctx.executed_evals(True)
            ctx.executed_evals(False)
            corners = r.nx * r.ny
            do_dense = corners <= a.dense_max
            band_ms, dense_ms = [], []
            for _ in range(a.reps):
                band_ms.append(timed(lambda: ctx.swept_contour(T, co, h, iso))[0])
                if do_dense:
                    ms, o = timed(lambda: dense_contour(ctx, T, co, r, iso))
                    dense_ms.append(ms)
            same = None
            if do_dense:
                same = bool(np.array_equal(r.vertices.view(np.uint64), o.vertices.view(np.uint64)) and np.array_equal(r.segments, o.segments)
                            and np.array_equal(r.triangles, o.triangles))
                assert same, (name, h)
            rec = dict(scene=name, N=int(len(T)), D=float(np.sum(T)), h=h, iso=iso, nx=r.nx, ny=r.ny, corners=corners,
                       evaluated=r.n_evaluated, executed_evals=int(evals), launches=int(launches), V=len(r.vertices),
                       S=len(r.segments), F=len(r.triangles), clipped=r.clipped, band_ms=float(np.median(band_ms)),
                       dense_ms=float(np.median(dense_ms)) if do_dense else None, dense_identical=same)
            print(json.dumps(rec), flush=True)
            lines.append(rec)
        ctx.close()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(json.dumps(dict(card=card)), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            for rec in lines:
                fh.write(json.dumps(rec) + "\n")
            fh.write(json.dumps(dict(card=card)) + "\n")


if __name__ == "__main__":
    main()
