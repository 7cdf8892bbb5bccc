"""The reference's OWN outer solver (the prebuilt LMBM binary, src/utils/include/utils/lmbm.so, default parameters of
back_end_optimizer.cpp:29) driving THIS library's cost callback on the GPU: `svsdf_evaluate` has the lmbm_evaluate_t
signature (lmbm.h:206-209), so its address is handed to lmbm_optimize as is — no Python in the loop (INTEGRATION.md §2).

    python tests/tools/run_lmbm_gpu.py [--points 400 --pieces 8 --clearance 2.6 --seed-map 777 --max-evals 400] [--trace out.npz]
                                       [--lib PATH]

By default it needs oracle/_ref/lmbm.so (copied there by __graft_entry__.build() where the reference checkout is present;
git-ignored) and a libgfortran.so.5 (scipy bundles one; symlinked into oracle/_ref/), and re-executes itself with
LD_LIBRARY_PATH set.  --lib runs any other library exporting lmbm::lmbm_optimize instead (tests/cpp/lmbm_standin.cpp).  --trace records every (x, f) through a thin Python wrapper instead (slower; used by the tests).
Prints one JSON line."""
import argparse
import ctypes as C
import glob
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REFDIR = os.path.join(ROOT, "oracle", "_ref")
LMBM = os.path.join(REFDIR, "lmbm.so")
SYM = "_ZN4lmbm13lmbm_optimizeEiPdS0_PFdPvPKdS0_iES1_PFiS1_S3_iEPNS_16lmbm_parameter_tE"  # lmbm::lmbm_optimize (lmbm.h:214-221)


def ensure_loader_path():
    if os.environ.get("SVSDF_LMBM_REEXEC") == "1":
        return
    link = os.path.join(REFDIR, "libgfortran.so.5")
    extra = [REFDIR]
    if not os.path.exists(link):  # dangling or missing: look for scipy's bundled copy
        import scipy

        cand = sorted(glob.glob(os.path.join(os.path.dirname(scipy.__file__), "..", "scipy.libs", "libgfortran-*.so.5*")))
        if cand:
            os.makedirs(REFDIR, exist_ok=True)
            if os.path.lexists(link):
                os.remove(link)
            os.symlink(os.path.abspath(cand[0]), link)
    if os.path.exists(link):
        extra.append(os.path.dirname(os.path.realpath(link)))  # its libquadmath sits next to it
    env = dict(os.environ, SVSDF_LMBM_REEXEC="1", LD_LIBRARY_PATH=":".join(extra + [os.environ.get("LD_LIBRARY_PATH", "")]))
    os.execve(sys.executable, [sys.executable] + sys.argv, env)


class LmbmParam(C.Structure):  # lmbm.h:15-174 (values below are the struct's member initialisers)
    _fields_ = [("timeout", C.c_float), ("bundle_size", C.c_int), ("ini_corrections", C.c_int), ("max_corrections", C.c_int),
                ("exponent_distmeasure", C.c_int), ("max_iterations", C.c_int), ("max_evaluations", C.c_int), ("past", C.c_int),
                ("verbose", C.c_int), ("update_method", C.c_int), ("scaling_strategy", C.c_int), ("delta_past", C.c_double),
                ("f_rel_eps", C.c_double), ("f_lower_bound", C.c_double), ("terminate_param1", C.c_double), ("terminate_param2", C.c_double),
                ("distance_measure", C.c_double), ("sufficient_dec", C.c_double), ("max_stepsize", C.c_double)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=400)
    ap.add_argument("--pieces", type=int, default=8)
    ap.add_argument("--clearance", type=float, default=2.6)
    ap.add_argument("--seed-map", type=int, default=777)
    ap.add_argument("--max-evals", type=int, default=400)
    ap.add_argument("--trace", default=None)
    ap.add_argument("--lib", default=None, help="library exporting lmbm::lmbm_optimize (default: oracle/_ref/lmbm.so)")
    ap.add_argument("--plugin", action="store_true", help="go through the library's own plug-in (svsdf_set_lmbm_library + svsdf_optimize) "
                                                          "instead of calling lmbm_optimize from here")
    args = ap.parse_args()
    global LMBM
    if args.lib:  # a self-contained library: no Fortran runtime to find
        LMBM = os.path.abspath(args.lib)
    elif not os.path.exists(LMBM):
        print(json.dumps({"unavailable": "oracle/_ref/lmbm.so not present (copied there only where the reference checkout is present)"}))
        return
    else:
        ensure_loader_path()
    import numpy as np

    sys.path.insert(0, ROOT)
    from implicit_svsdf_planner_b200 import api, scenes

    sc = scenes.make_scene("star", args.pieces, args.points, clearance=args.clearance, seed_map=args.seed_map)
    opt = api.TrajOptimizer("star", weight_p=sc.weight_p, safety_hor=sc.safety_hor, rho=sc.rho, strict_fp=True)
    opt.parallel_points = sc.points
    opt.setConditions(sc.init_s, sc.final_s, sc.N)
    f0, _ = opt.costFunction(sc.x0)
    if args.plugin:
        # the context loads its own private instance of the library and svsdf_optimize runs it on svsdf_evaluate (what a batch worker does)
        lp = api.lmbm_default_params(max_evaluations=args.max_evals)
        opt.ctx.set_lmbm_library(LMBM, lp)
        t0 = time.perf_counter()
        rc, x, T, b, st = opt.ctx.optimize(sc.init_s, sc.final_s, sc.x0, sc.N, None)
        dt = time.perf_counter() - t0
        f_end, _ = opt.costFunction(x)
        print(json.dumps({"solver": "reference lmbm.so through svsdf_set_lmbm_library", "points": int(sc.P), "pieces": int(sc.N),
                          "lmbm_return": int(st["status"]), "optimize_return": int(rc), "f_start": float(f0), "f_final": float(st["final_cost"]),
                          "f_at_final_x": float(f_end), "iterations": int(st["iterations"]), "evaluations": int(st["evaluations"]), "seconds": dt}), flush=True)
        return
    L = C.CDLL(LMBM)
    lmbm_optimize = getattr(L, SYM)
    lmbm_optimize.restype = C.c_int
    dp = C.POINTER(C.c_double)
    EVAL = C.CFUNCTYPE(C.c_double, C.c_void_p, dp, dp, C.c_int)
    PROG = C.CFUNCTYPE(C.c_int, C.c_void_p, dp, C.c_int)
    iters = []
    prog = PROG(lambda _i, _x, k: (iters.append(k), 0)[1])
    xs, fs = [], []
    if args.trace:
        def ev(_inst, xp, gp, n):
            x = np.ctypeslib.as_array(xp, shape=(n,)).copy()
            f, g = opt.costFunction(x)
            np.ctypeslib.as_array(gp, shape=(n,))[:] = g
            xs.append(x); fs.append(f)
            return float(f)
        evaluate, instance = EVAL(ev), None
    else:
        evaluate = C.cast(api.lib().svsdf_evaluate, EVAL)  # the library's C entry point itself
        instance = opt.ctx.h
    p = LmbmParam(300.0, 2, 7, 15, 2, 10000, 20000, 10, -1, 0, 0, 1.0e-8, 1.0e+4, -1.0e+60, 1.0e-6, 1.0e-6, 0.5, 1.0e-4, 1.5)
    p.max_evaluations = args.max_evals
    x = sc.x0.copy()
    fx = C.c_double()
    t0 = time.perf_counter()
    ret = lmbm_optimize(C.c_int(x.size), x.ctypes.data_as(dp), C.byref(fx), evaluate, instance, prog, C.byref(p))
    dt = time.perf_counter() - t0
    f_end, _ = opt.costFunction(x)
    n_it = (max(iters) if iters else 0)
    if args.trace:
        np.savez_compressed(args.trace, xs=np.array(xs), fs=np.array(fs), final_x=x, final_f=fx.value, lmbm_return=ret)
    print(json.dumps({"solver": "reference lmbm.so", "callback": "svsdf_evaluate (GPU)" if not args.trace else "svsdf_evaluate via python trace wrapper",
                      "points": int(sc.P), "pieces": int(sc.N), "lmbm_return": int(ret), "f_start": float(f0), "f_final": float(fx.value),
                      "f_at_final_x": float(f_end), "iterations": int(n_it), "evaluations_traced": len(fs) if args.trace else None,
                      "seconds": dt, "iters_per_s": n_it / dt if dt > 0 else None}), flush=True)


if __name__ == "__main__":
    main()
