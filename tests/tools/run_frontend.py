"""K5 measurement: configuration-space obstacle map (kernelConv for every yaw kernel and cell) of the batch mode's map
(60 m at 0.025 m = 2400 x 2400 cells, 18 yaw kernels of 17 x 17) on one GPU, next to the oracle's restatement of the
reference's kernelConv<true> on the host cores (a crop, scaled).  Prints one JSON line."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
from implicit_svsdf_planner_b200 import api, batch
from oracle import oracle_py as O

ks, K, res = 17, 18, 0.025
gm = batch.make_random_map(extent=60.0, res=res, density=float(os.environ.get("SVSDF_DENSITY", "0.27")), seed=20240502)
X, Y = gm.shape
ctx = api.Context("star")
t0 = time.perf_counter(); ctx.front_init(ks, K, res, 0.0); t_init = time.perf_counter() - t0
ctx.set_map(batch.pack_map_kernel(gm.occ, ks), X, Y, ks, (0.0, 0.0), res)
for _ in range(3):
    ctx.front_cspace(X, Y, fetch=False)
ms = [ctx.front_cspace(X, Y, fetch=False)[1] for _ in range(20)]
ms_med = float(np.median(ms))
W = (Y + 31) // 32
out_bytes = K * X * W * 4
in_bytes = (X + ks - 1) * ((Y + ks - 1 + 7) // 8)
peaks = {}
pp = os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "MEASURED_PEAKS.json")
if os.path.exists(pp):
    peaks = json.load(open(pp))
hbm = peaks.get("hbm_gbs", 3350.0)
# CPU: the oracle's kernelConv<true> over a crop, all host threads (OpenMP), scaled by cell count
n = 400
crop = gm.occ[:n, :n]
t0 = time.perf_counter(); O.cspace("star", crop, ks, K, res, 0.0, variant="byte"); t_cpu = time.perf_counter() - t0
cells = K * X * Y
rec = {"kernel": "k_cspace", "map_cells": [X, Y], "yaw_kernels": K, "kernel_size": ks, "gpu_ms": ms_med, "gpu_ms_min": float(min(ms)),
       "kernel_conv_per_s_gpu": cells / (ms_med * 1e-3), "front_init_s": t_init,
       "roofline": {"bound": "hbm", "algorithmic_bytes": out_bytes + in_bytes, "achieved": (out_bytes + in_bytes) / (ms_med * 1e-3) / 1e9,
                    "peak": hbm, "unit": "GB/s", "frac": (out_bytes + in_bytes) / (ms_med * 1e-3) / 1e9 / hbm,
                    "peak_source": "MEASURED_PEAKS.json" if peaks else "H100 SXM data sheet, 3350 GB/s"},
       "cpu": {"kernel_conv_per_s": K * n * n / t_cpu, "threads": O.num_procs(), "sample": f"{n} x {n} crop, {K} kernels, oracle kernelConv<true> restatement"},
       "speedup": (cells / (ms_med * 1e-3)) / (K * n * n / t_cpu)}
# node expansion (AstarPathSearcher::process neighbour loop) for 4096 nodes at once — one node per problem of the batch mode —
# on a front-end grid like the reference's (occupancy_resolution 1.0, 60 x 60 cells)
rng = np.random.default_rng(7)
occ2 = rng.random((60, 60)) < 0.03
ctx2 = api.Context("star")
ctx2.front_init(17, 18, 1.0, 0.0)
ctx2.set_map(batch.pack_map_kernel(occ2, 17), 60, 60, 17, (0.0, 0.0), 1.0)
ij = np.stack([rng.integers(0, 60, 4096), rng.integers(0, 60, 4096)], axis=1)
fy = rng.uniform(-3.14, 3.14, 4096)
ctx2.front_expand(ij, fy)
t0 = time.perf_counter()
for _ in range(10):
    ok, cy, parts = ctx2.front_expand(ij, fy)
t_gpu = (time.perf_counter() - t0) / 10
t0 = time.perf_counter(); O.expand_nodes("star", occ2, ij, fy, map_res=1.0); t_cpu2 = time.perf_counter() - t0
rec["expand"] = {"nodes": 4096, "gpu_ms_e2e": 1e3 * t_gpu, "cpu_ms": 1e3 * t_cpu2, "cpu_threads": O.num_procs(), "speedup": t_cpu2 / t_gpu,
                 "pass_rate": float(ok.mean()), "note": "host buffers in and out (svsdf_front_expand), 9 neighbours per node"}
# batch A*: 1024 start/goal problems in lock-step (svsdf_front_astar) vs the oracle's AstarPathSearch per problem (OpenMP over problems)
occ3 = rng.random((60, 60)) < 0.005
ctx3 = api.Context("star")
ctx3.front_init(17, 18, 1.0, 0.0)
ctx3.set_map(batch.pack_map_kernel(occ3, 17), 60, 60, 17, (0.0, 0.0), 1.0)
npb = int(os.environ.get("SVSDF_ASTAR_PROBLEMS", "1024"))
st = rng.uniform(1.0, 59.0, size=(npb, 2)); go = rng.uniform(1.0, 59.0, size=(npb, 2))
ctx3.front_astar(st[:8], go[:8])
t0 = time.perf_counter(); paths, ex, rounds = ctx3.front_astar(st, go); t_gpu = time.perf_counter() - t0
t0 = time.perf_counter(); paths_o, ex_o = O.astar("star", occ3, st, go, map_res=1.0); t_cpu3 = time.perf_counter() - t0
same = bool(np.array_equal(ex, ex_o) and all((a is None) == (b is None) and (a is None or np.array_equal(a, b)) for a, b in zip(paths, paths_o)))
rec["astar"] = {"problems": npb, "found": int(sum(p is not None for p in paths)), "expansions": int(ex.sum()), "lockstep_rounds": int(rounds),
                "gpu_s": t_gpu, "cpu_s": t_cpu3, "cpu_threads": O.num_procs(), "speedup": t_cpu3 / t_gpu, "identical_to_oracle": same,
                "problems_per_s_gpu": npb / t_gpu}
print(json.dumps(rec))
