"""Back-end measurement: the lock-step back end on the host, its machines advanced round by round (svsdf_optimize_lockstep), against
the device back end (svsdf_optimize_device) on the inputs of run_plan_batch.py's four workloads (star scene and grid60 at n = 256 and
1024), taken from plan.plan_batch(back_end=False).  The two arms alternate in one process, three runs each, on one context; every problem's result must be
identical between them (status, iterations, evaluations, x, T, coefficients, cost at the start, final cost) or the script exits non-zero.
Prints one JSON line per workload: median wall seconds of each arm, rounds and launches per round, and per round the device time of the
evaluation kernels, of the back-end kernels and the remainder (host work, copies and gaps); with the GPU's name, power limit and max SM
clock.

    python tests/tools/run_optimize_device.py [--sizes 256,1024] [--scenes star,grid60] [--runs 3]
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402
import run_plan_batch as W  # noqa: E402  (the workloads, the context and the GPU query)

from implicit_svsdf_planner_b200 import api, plan  # noqa: E402

KEYS = ("status", "iterations", "evaluations", "solver_status")
BITS = ("x", "T", "coeffs", "cost_at_start", "final_cost")


def identical(a, b):
    for g, r in zip(a, b):
        if any(g[k] != r[k] for k in KEYS):
            return False
        if any(not np.array_equal(np.asarray(g[k], dtype=np.float64).view(np.uint64), np.asarray(r[k], dtype=np.float64).view(np.uint64))
               for k in BITS):
            return False
    return len(a) == len(b)


def run_arm(ctx, fn, probs, params):
    l0 = ctx.kernel_launches()
    t0 = time.perf_counter()
    res, rounds = fn(probs, params)
    wall = time.perf_counter() - t0
    ev, be = ctx.round_times()
    return res, dict(wall=wall, rounds=rounds, launches=ctx.kernel_launches() - l0, eval_ms=ev, backend_ms=be)


def summary(runs):
    med = sorted(runs, key=lambda r: r["wall"])[len(runs) // 2]
    R = max(med["rounds"], 1)
    return dict(wall_s=statistics.median(r["wall"] for r in runs), rounds=med["rounds"], launches_per_round=med["launches"] / R,
                round_ms=1e3 * med["wall"] / R, round_eval_kernels_ms=med["eval_ms"] / R, round_backend_kernels_ms=med["backend_ms"] / R,
                round_rest_ms=(1e3 * med["wall"] - med["eval_ms"] - med["backend_ms"]) / R)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="256,1024")
    ap.add_argument("--scenes", default="star,grid60")
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    info = W.gpu_info()
    params = api.default_lbfgs_params(mem_size=16, past=3, delta=1e-6, g_epsilon=0.0, max_iterations=0, min_step=1e-32)
    ok = True
    for name in a.scenes.split(","):
        cmap, kw = W.star_scene() if name == "star" else W.grid60_scene()
        for n in (int(s) for s in a.sizes.split(",")):
            st, go = W.pairs(cmap, n, 1000 + n)
            ctx = W.new_ctx()
            inputs = [r for r in plan.plan_batch(ctx, cmap, st, go, back_end=False, **kw) if r["ok"]]
            probs = [dict(N=r["N"], init_s=r["init_s"], final_s=r["final_s"], x0=r["x0"], points=r["points"]) for r in inputs]
            arms = {"lockstep": (ctx.optimize_lockstep, []), "device": (ctx.optimize_device, [])}
            first = {}
            for _ in range(a.runs):
                for arm, (fn, runs) in arms.items():
                    res, m = run_arm(ctx, fn, probs, params)
                    runs.append(m)
                    first.setdefault(arm, res)
                    ok &= identical(res, first["lockstep"])
            ctx.close()
            rec = {"scene": name, "n": n, "problems": len(probs), "identical": bool(ok)}
            for arm, (_, runs) in arms.items():
                rec[arm] = summary(runs)
            rec["speedup"] = rec["lockstep"]["wall_s"] / rec["device"]["wall_s"]
            rec.update(info)
            print(json.dumps(rec), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
