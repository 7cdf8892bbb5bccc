"""Times config 2 (star, N = 8, 200 000 points) rigid against the reference's example deformation schedule on one GPU and
prints one JSON line per case: ms per cost + gradient evaluation (fast build, device-resident points, CUDA events), the
per-kernel split, and an L-BFGS run (iterations, evaluations, seconds).  Also records the GPU name, power limit and SM clock.

    python tests/tools/run_scale.py [--lbfgs 60]
"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from implicit_svsdf_planner_b200 import api, scenes  # noqa: E402


def gpu_info():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:  # informative only
        return f"unavailable ({e})"


def run(case, sc, co, scale, lbfgs_iters):
    ctx = api.Context("star", weight_p=sc.weight_p, safety_hor=sc.safety_hor, rho=sc.rho, strict_fp=False)
    if scale:
        ctx.set_scale(**api.EXAMPLE_SCALE)
    ctx.set_points(sc.points)
    ctx.cost_grad_device(sc.T, co, repeats=3, fetch=False)
    samples = [ctx.cost_grad_device(sc.T, co, repeats=10)[0] for _ in range(5)]
    ms, out = ctx.cost_grad_device(sc.T, co, repeats=10)
    rec = dict(case=case, P=sc.P, N=sc.N, ms_per_eval_median=sorted(samples)[2], ms_per_eval_min=min(samples),
               ms_per_eval_max=max(samples), kernel_ms=ctx.last_kernel_ms(), n_inside=int(out[-1]), cost=float(out[0]))
    if lbfgs_iters:
        params = api.default_lbfgs_params(mem_size=16, past=3, delta=1e-6, g_epsilon=0.0, max_iterations=lbfgs_iters, min_step=1e-32)
        rc, x, T, b, st = ctx.optimize(sc.init_s, sc.final_s, sc.x0, sc.N, params)
        rec["lbfgs"] = dict(status=st["status"], iterations=st["iterations"], evaluations=st["evaluations"], seconds=st["seconds"],
                            final_cost=st["final_cost"])
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    it = int(sys.argv[sys.argv.index("--lbfgs") + 1]) if "--lbfgs" in sys.argv else 60
    print(json.dumps(dict(gpu=gpu_info())), flush=True)
    sc = scenes.make_scene("star", 8, 200_000)
    co = sc.coeffs_colmajor()
    run("rigid", sc, co, False, it)
    run("example_schedule", sc, co, True, it)
    run("rigid_again", sc, co, False, 0)
