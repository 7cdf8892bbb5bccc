"""Pose-sampled obstacle penalty measurement (svsdf_set_pose_penalty).

0. k_pose's own time (torch.profiler, CUDA activities) for one trajectory of config 2's size (8 pieces, star shape) on the star map at
   star.yaml's values: svsdf_pose_penalty_eval repeated, the mean k_pose duration.
1. Device back end (svsdf_optimize_device) on the problems of star-scene start / goal pairs that reach the back end, the penalty off
   against on (star.yaml's values), alternating: wall seconds, rounds, launches per round and per round the device time of the
   back-end kernels (svsdf_round_times' backend_ms / rounds: k_backend_blob, k_pose and k_backend_backward).
2. plan.plan_batch(certify=True) on the star scene and on grid60 with the coords.txt pairs, in three variants: SVSDF only (today),
   pose only (the SVSDF term's weight_p set to 0) and both.  Per run: back-end seconds, rounds, collision-free plans.
Prints one JSON line per measurement, with the GPU's name, power limit and max SM clock.

    python tests/tools/run_pose_penalty.py [--n 1024] [--runs 2] [--plan-n 256 1024]
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402
import run_dynamics as D  # noqa: E402  (back-end inputs)
import run_plan_batch as W  # noqa: E402  (scenes, contexts and the GPU query)

from implicit_svsdf_planner_b200 import api, plan, scenes  # noqa: E402

PARAMS = D.PARAMS


def device_arm(ctx, probs):
    n0 = ctx.kernel_launches()
    t0 = time.perf_counter()
    res, rounds = ctx.optimize_device(probs, PARAMS)
    sec = time.perf_counter() - t0
    ev, be = ctx.round_times()
    return dict(seconds=sec, rounds=rounds, launches_per_round=(ctx.kernel_launches() - n0) / rounds, eval_ms_per_round=ev / rounds,
                backend_ms_per_round=be / rounds, iterations=int(sum(r["iterations"] for r in res)))


def kernel_time(cmap, kw, pose, reps=200):
    import torch
    from torch.profiler import ProfilerActivity, profile

    ctx = W.new_ctx()
    X, Y, Z = cmap.occ.shape
    ctx.set_map3d(plan.pack_map_kernel3d(cmap.occ, kw["kernel_size"]), X, Y, Z, kw["kernel_size"], cmap.boundary_min, cmap.res)
    sc = scenes.make_scene("star", 8, 0)
    b, *_ = api.minco_forward(sc.init_s, sc.final_s, sc.q, sc.T)
    co = np.ascontiguousarray(b.T).reshape(-1)
    for _ in range(10):
        ctx.pose_penalty(sc.T, co, pose)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ctx.pose_penalty(sc.T, co, pose)
        torch.cuda.synchronize()
    us = [e.device_time for e in prof.events() if "k_pose" in e.name]
    ctx.close()
    return dict(samples=8 * (pose.integralIntervs + 1), launches=len(us), k_pose_us_mean=float(np.mean(us)) if us else None,
                k_pose_us_median=float(np.median(us)) if us else None)


def variant_ctx(name):
    y = scenes.YAML
    ctx = api.Context("star", weight_p=0.0 if name == "pose_only" else y["weight_p"], safety_hor=y["safety_hor"], rho=y["rho"])
    if name != "svsdf_only":
        ctx.set_pose_penalty(api.yaml_pose_penalty(y))
    return ctx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--plan-n", type=int, nargs="+", default=[256, 1024])
    a = ap.parse_args()
    info = W.gpu_info()
    pose = api.yaml_pose_penalty(scenes.YAML)

    cmap, kw = W.star_scene()
    print(json.dumps(dict(what="k_pose per evaluation, 8 pieces, star map", **kernel_time(cmap, kw, pose), **info)), flush=True)
    probs = D.back_end_inputs(cmap, kw, a.n, 1)
    ctx = W.new_ctx()
    X, Y, Z = cmap.occ.shape
    ctx.set_map3d(plan.pack_map_kernel3d(cmap.occ, kw["kernel_size"]), X, Y, Z, kw["kernel_size"], cmap.boundary_min, cmap.res)
    device_arm(ctx, probs[:8])  # warm-up
    arms = {"off": [], "on": []}
    for _ in range(a.runs):
        for name in ("off", "on"):
            ctx.set_pose_penalty(None if name == "off" else pose)
            arms[name].append(device_arm(ctx, probs))
    ctx.close()
    rec = dict(what="device back end, star scene", problems=len(probs), **info)
    for name, runs in arms.items():
        rec[name] = {k: statistics.median(r[k] for r in runs) for k in runs[0]}
    print(json.dumps(rec), flush=True)

    grid, gkw = W.grid60_scene()
    for n in a.plan_n:
        sg = scenes.make_batch_problems(n)
        for scene_name, cm, kk, (st, go) in (("star", cmap, kw, W.pairs(cmap, n, 2)), ("grid60", grid, gkw, (sg[:, :2], sg[:, 2:]))):
            st, go = np.asarray(st), np.asarray(go)
            for name in ("svsdf_only", "pose_only", "both"):
                s = {}
                c = variant_ctx(name)
                out = plan.plan_batch(c, cm, st, go, certify=True, stats=s, **kk)
                c.close()
                done = [r for r in out if r and "T" in r]
                print(json.dumps(dict(what=f"plan_batch certify, {scene_name}, n {n}, {name}", plans=len(done), back_s=s.get("back_s"),
                                      rounds=s.get("rounds"), iterations=int(sum(r["iterations"] for r in done)),
                                      collision_free=int(sum(r["clearance"]["collision_free"] for r in done)), **info)), flush=True)


if __name__ == "__main__":
    main()
