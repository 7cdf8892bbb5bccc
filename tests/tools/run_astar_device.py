"""Device A* measurement: svsdf_front_astar_device (whole searches in one launch) next to the lock-step svsdf_front_astar (one
expand launch, two copies and a host open-list pass per round) on the same searches, in the same process.

Workloads: the run_frontend.py scene (star, 60 x 60 cells at resolution 1.0, 17 x 17 kernels, 18 yaws) at obstacle densities 0.005
and 0.03 with 1024 and 4096 seeded start / goal pairs, and the single search of the reference's star scene (tests/golden/
map_star_pcd.npz, as tests/test_gpu_plan.py builds it).  Per workload: both entries warmed up, then timed alternately (--reps
times each; every call ends in a stream synchronise), outputs checked identical (paths, lengths, expansion counts).  Prints one
JSON line per workload, with the GPU's name, power limit and max SM clock."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from implicit_svsdf_planner_b200 import api, batch, plan, scenes  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = (v.strip() for v in r.stdout.splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def identical(a, b):
    pa, ea = a[0], a[1]
    pb, eb = b[0], b[1]
    return bool(np.array_equal(ea, eb) and all((x is None) == (y is None) and (x is None or np.array_equal(x, y)) for x, y in zip(pa, pb)))


def measure(ctx, st, go, max_path, reps):
    lock = ctx.front_astar(st, go, max_path)  # warm-up of both entries (and the device pool)
    dev = ctx.front_astar_device(st, go, max_path)
    t_lock, t_dev, ms_dev = [], [], []
    for _ in range(reps):
        t0 = time.perf_counter(); lock = ctx.front_astar(st, go, max_path); t_lock.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); dev = ctx.front_astar_device(st, go, max_path); t_dev.append(time.perf_counter() - t0)
        ms_dev.append(dev[3])
    return {"searches": len(st), "found": int(sum(p is not None for p in dev[0])), "expansions": int(dev[1].sum()),
            "max_expansions_one_search": int(dev[1].max()), "lockstep_rounds": int(lock[2]),
            "lockstep_s_median": float(np.median(t_lock)), "lockstep_s_min": float(min(t_lock)),
            "device_s_median": float(np.median(t_dev)), "device_s_min": float(min(t_dev)),
            "device_kernel_ms_median": float(np.median(ms_dev)), "speedup_median": float(np.median(t_lock) / np.median(t_dev)),
            "identical": identical(lock, dev), "status_counts": {str(s): int(c) for s, c in zip(*np.unique(dev[2], return_counts=True))}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--problems", default="1024,4096")
    ap.add_argument("--densities", default="0.005,0.03")
    a = ap.parse_args()
    info = gpu_info()
    ok = True
    for dens in (float(d) for d in a.densities.split(",")):
        rng = np.random.default_rng(7)
        occ = rng.random((60, 60)) < dens
        ctx = api.Context("star")
        ctx.front_init(17, 18, 1.0, 0.0)
        ctx.set_map(batch.pack_map_kernel(occ, 17), 60, 60, 17, (0.0, 0.0), 1.0)
        for npb in (int(p) for p in a.problems.split(",")):
            prng = np.random.default_rng(npb)
            st, go = prng.uniform(1.0, 59.0, size=(npb, 2)), prng.uniform(1.0, 59.0, size=(npb, 2))
            rec = {"workload": f"star 60x60 density {dens} x {npb}", **measure(ctx, st, go, 1024, a.reps), **info}
            ok &= rec["identical"]
            print(json.dumps(rec), flush=True)
        ctx.close()
    g = np.load(os.path.join(ROOT, "tests", "golden", "map_star_pcd.npz"))
    res, ks = float(g["occupancy_resolution"]), int(g["kernel_size"])
    cmap = plan.gridmap3d_from_cloud(g["points"], res, int(g["sta_threshold"]))
    X, Y, Z = cmap.occ.shape
    ctx = api.Context("star", weight_p=scenes.YAML["weight_p"], safety_hor=scenes.YAML["safety_hor"], rho=scenes.YAML["rho"])
    ctx.set_map3d(plan.pack_map_kernel3d(cmap.occ, ks), X, Y, Z, ks, cmap.boundary_min, res)
    ctx.front_init(ks, 18, res, 0.0)
    rec = {"workload": f"reference star scene ({X} x {Y} cells), one search",
           **measure(ctx, g["start"][:2].reshape(1, 2), g["end"][:2].reshape(1, 2), 4096, a.reps), **info}
    ok &= rec["identical"]
    print(json.dumps(rec), flush=True)
    ctx.close()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
