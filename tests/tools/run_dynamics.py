"""Dynamics-penalty measurement (svsdf_set_dynamics).

1. Device back end (svsdf_optimize_device) on the problems of 1024 star-scene start / goal pairs that reach the back end
   (plan.plan_batch(back_end=False) inputs), dynamics off
   against on (star.yaml's limits), alternating, three runs each: total wall seconds, rounds, and per round the device time of the
   back-end kernels (svsdf_round_times' backend_ms / rounds, k_backend_backward with k_backend_blob and k_backend_init).
2. plan.plan_batch(certify=True) on the star scene and on grid60 with the coords.txt pairs: without dynamics, with star.yaml's limits
   and with vmax = 1 m/s.  Per run: plans over the limit (sampled, before = the same plans without the penalty), median and
   maximum v_peak, back-end iterations and seconds, collision-free count.
Prints one JSON line per measurement, with the GPU's name, power limit and max SM clock.

    python tests/tools/run_dynamics.py [--n 1024] [--runs 3] [--plan-n 256]
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402
import run_plan_batch as W  # noqa: E402  (scenes, contexts and the GPU query)

from implicit_svsdf_planner_b200 import api, plan, scenes  # noqa: E402

PARAMS = api.default_lbfgs_params(mem_size=16, past=3, delta=1e-6, g_epsilon=0.0, max_iterations=0, min_step=1e-32)


def back_end_inputs(cmap, kw, n, seed):
    st, go = W.pairs(cmap, n, seed)
    ctx = W.new_ctx()
    res = plan.plan_batch(ctx, cmap, st, go, back_end=False, **kw)
    ctx.close()
    return [dict(N=r["N"], init_s=r["init_s"], final_s=r["final_s"], x0=r["x0"], points=r["points"]) for r in res if r and "x0" in r]


def device_arm(ctx, probs):
    t0 = time.perf_counter()
    res, rounds = ctx.optimize_device(probs, PARAMS)
    sec = time.perf_counter() - t0
    ev, be = ctx.round_times()
    return dict(seconds=sec, rounds=rounds, eval_ms_per_round=ev / rounds, backend_ms_per_round=be / rounds,
                iterations=int(sum(r["iterations"] for r in res)))


def over(results, dyn):
    n = 0
    for r in results:
        rep = plan.dynamics_report(dyn, r["T"], r["coeffs"])
        n += not rep["within_limits"]
    return n


def plan_summary(out, dyn, stats):
    done = [r for r in out if r and "T" in r]
    peaks = np.array([plan.dynamics_report(dyn, r["T"], r["coeffs"])["v_peak"] for r in done])
    return dict(plans=len(done), over_limit=over(done, dyn), v_peak_median=float(np.median(peaks)) if len(peaks) else None,
                v_peak_max=float(peaks.max()) if len(peaks) else None, iterations=int(sum(r["iterations"] for r in done)),
                back_s=stats.get("back_s"), collision_free=int(sum(r["clearance"]["collision_free"] for r in done)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--plan-n", type=int, default=256)
    a = ap.parse_args()
    info = W.gpu_info()
    yaml = api.yaml_dynamics(scenes.YAML).as_dict()

    cmap, kw = W.star_scene()
    probs = back_end_inputs(cmap, kw, a.n, 1)
    ctx = W.new_ctx()
    device_arm(ctx, probs[:8])  # warm-up
    arms = {"off": [], "on": []}
    for _ in range(a.runs):
        for name in ("off", "on"):
            ctx.set_dynamics(None if name == "off" else yaml)
            arms[name].append(device_arm(ctx, probs))
    ctx.close()
    rec = dict(what="device back end, star scene", problems=len(probs), **info)
    for name, runs in arms.items():
        rec[name] = {k: statistics.median(r[k] for r in runs) for k in runs[0]}
    print(json.dumps(rec), flush=True)

    grid, gkw = W.grid60_scene()
    sg = scenes.make_batch_problems(a.plan_n)
    for scene_name, cm, kk, (st, go) in (("star", cmap, kw, W.pairs(cmap, a.plan_n, 2)), ("grid60", grid, gkw, (sg[:, :2], sg[:, 2:]))):
        st, go = np.asarray(st), np.asarray(go)
        base_stats = {}
        c0 = W.new_ctx()
        base = plan.plan_batch(c0, cm, st, go, certify=True, stats=base_stats, **kk)
        c0.close()
        for label, dyn in (("yaml", yaml), ("vmax_1", dict(yaml, vmax=1.0))):
            s = {}
            c1 = W.new_ctx()
            c1.set_dynamics(dyn)
            out = plan.plan_batch(c1, cm, st, go, certify=True, stats=s, **kk)
            c1.close()
            print(json.dumps(dict(what=f"plan_batch certify, {scene_name}, limits {label}", limits=dyn, before=plan_summary(base, dyn, base_stats),
                                  after=plan_summary(out, dyn, s), **info)), flush=True)


if __name__ == "__main__":
    main()
