"""Where the batched k_outer's warp-cycles go: the descent's lane efficiency and the share of every phase, from counters in the kernel.

    python scripts/outer_phase_stats.py [--build-dir DIR] [--no-build] [--chunk N] [--configs 2 3]

Builds the strict kernel unit with -DSVSDF_PHASE_STATS (svsdf_kernels.cuh) into DIR (default: a temporary directory), links it
with the product's other objects into DIR/libsvsdf_phase_stats.so and runs one cost-and-gradient evaluation of BASELINE config 2
(star, 8 pieces, 200 000 points) and config 3 (sdHorseshoe, 16 pieces, 500 000 points) on it.  The product library is not touched.
--no-build uses the library already in DIR (build on a machine without a GPU, run on one with).  --chunk N runs under
SVSDF_FORCE_OUTER_CHUNK = N (1: one descent pass per batch of a warp); without it the runtime picks the chunk.

One JSON line per config:
  descent_lane_efficiency   useful / issued descent lane-evaluations (a warp issues 64 per engine iteration, whatever its groups do)
  share_seed, share_descent, share_wait_after_descent, share_epilogue
                            warp-cycles (clock64) of the seed scan (up to the barrier that opens the queue), the descent, the wait at
                            the barrier after it, and the gradient + epilogue + accumulation, over their sum, all warps of the grid
A diagnostic: it needs a GPU and fails without one.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = {"2": ("star", 8, 200_000, 2.75), "3": ("sdHorseshoe", 16, 500_000, 2.15)}  # tests/tools/run_configs.py
LIB = "libsvsdf_phase_stats.so"


def build(out_dir):
    from implicit_svsdf_planner_b200 import build as pb

    pb.build()  # the other units' objects
    unit = next(u for u in pb.UNITS if u[0] == "svsdf_kernels_strict.cu")
    obj = os.path.join(out_dir, "svsdf_kernels_strict_stats.o")
    subprocess.check_call([pb.NVCC, *pb.ARCH, *pb.COMMON, *unit[2], "-DSVSDF_PHASE_STATS", "-c", os.path.join(pb.CSRC, unit[0]), "-o", obj])
    objs = [obj if u is unit else os.path.join(pb.OBJDIR, u[1]) for u in pb.UNITS]
    subprocess.check_call([pb.NVCC, *pb.ARCH, "-shared", "-ccbin", "/usr/bin/g++", "-Xcompiler", "-fopenmp", "-o", os.path.join(out_dir, LIB),
                           *objs, "-lgomp"])


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--build-dir")
    ap.add_argument("--no-build", action="store_true")
    ap.add_argument("--chunk", type=int)
    ap.add_argument("--configs", nargs="+", default=["2", "3"], choices=sorted(CONFIGS))
    args = ap.parse_args()
    out_dir = args.build_dir or tempfile.mkdtemp(prefix="svsdf_phase_stats_")
    os.makedirs(out_dir, exist_ok=True)
    if not args.no_build:
        build(out_dir)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("outer_phase_stats: no GPU")
    from implicit_svsdf_planner_b200 import api, scenes

    api.LIB_PATH = os.path.join(out_dir, LIB)
    if args.chunk is None:
        os.environ.pop("SVSDF_FORCE_OUTER_CHUNK", None)
    else:
        os.environ["SVSDF_FORCE_OUTER_CHUNK"] = str(args.chunk)
    L = api.lib()
    L.svsdf_phase_stats_buffer.argtypes = [ctypes.c_void_p]
    prop = torch.cuda.get_device_properties(0)
    buf = torch.zeros(prop.multi_processor_count * 8 * 8 * 6, dtype=torch.int64, device="cuda")  # up to 8 CTAs per SM
    if L.svsdf_phase_stats_buffer(buf.data_ptr()) != 0:
        raise SystemExit("outer_phase_stats: cudaMemcpyToSymbol failed")
    for name in args.configs:
        shape, N, P, clearance = CONFIGS[name]
        sc = scenes.make_scene(shape, N, P, clearance=clearance)
        ctx = api.Context(shape, weight_p=sc.weight_p, safety_hor=sc.safety_hor, rho=sc.rho, strict_fp=True)
        ctx.set_points(sc.points)
        co = sc.coeffs_colmajor()
        ctx.cost_grad(sc.T, co)
        buf.zero_()
        torch.cuda.synchronize()
        ctx.cost_grad(sc.T, co)
        torch.cuda.synchronize()
        st = buf.cpu().numpy().reshape(-1, 6)
        st = st[st[:, 3] > 0]  # the warps that ran
        ctx.close()
        if not len(st):
            raise SystemExit(f"outer_phase_stats: config {name} did not run the batched schedule")
        issued, useful, seed, desc, wait, epi = (float(v) for v in st.sum(axis=0))
        total = seed + desc + wait + epi
        print(json.dumps(dict(
            config=name, shape=shape, N=N, P=P, chunk="runtime" if args.chunk is None else args.chunk, device=prop.name,
            warps=int(len(st)), descent_lane_efficiency=useful / issued, share_seed=seed / total, share_descent=desc / total,
            share_wait_after_descent=wait / total, share_epilogue=epi / total)), flush=True)


if __name__ == "__main__":
    main()
