"""Golden outputs of the host L-BFGS (host/lbfgs.hpp) and MINCO (host/minco.hpp) through the C ABI, recorded before both were
restated on flat storage for the device back end (svsdf_optimize_device).  tests/test_host_backend_golden.py requires the same bits.

    python tests/golden/make_backend_golden.py      (needs the built library, no GPU)

Stored in tests/golden/host_backend.npz:
  * svsdf_lbfgs_minimize on the Python callbacks of LBFGS_CASES, one per exit of the solver: every evaluated x in order, the returned
    x, status, final cost, iterations and evaluations;
  * svsdf_minco_forward / svsdf_minco_propagate on seeded inputs, N = 2 ... 64;
  * svsdf_mid_get_ori_traj on the cases of ref_mid.npz (the L-BFGS in its reference_patch mode)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from implicit_svsdf_planner_b200 import api  # noqa: E402
import make_mid_golden as mk  # noqa: E402  (the mid-end problem generator and its two parameter sets)

OUT = os.path.join(HERE, "host_backend.npz")
MINCO_N = (2, 3, 4, 5, 7, 8, 11, 16, 23, 32, 47, 63, 64)
MID_N = (2, 3, 6, 12)


def quadratic(x):
    a = np.arange(1.0, x.size + 1)
    c = np.linspace(-1.0, 2.0, x.size)
    return float(np.sum(a * (x - c) ** 2)), 2 * a * (x - c)


def rosenbrock(x):
    f = np.sum(100.0 * (x[1:] - x[:-1] ** 2) ** 2 + (1.0 - x[:-1]) ** 2)
    g = np.zeros_like(x)
    g[:-1] = -400.0 * x[:-1] * (x[1:] - x[:-1] ** 2) - 2.0 * (1.0 - x[:-1])
    g[1:] += 200.0 * (x[1:] - x[:-1] ** 2)
    return float(f), g


def abs_sum(x):
    """weighted sum of |A x - c| plus a small quadratic: kinks the minimiser sits on, never hit exactly"""
    c = np.array([0.1, -0.7, 0.33, 0.9]) * np.sqrt(2)
    w = np.array([1.0, 2.5, 0.7, 1.9])
    A = np.array([[1, 0.3, 0, 0.2], [0.1, 1, 0.4, 0], [0, 0.2, 1, 0.5], [0.3, 0, 0.1, 1]])
    r = A @ x - c
    return float(np.sum(w * np.abs(r)) + 0.05 * x @ x), A.T @ (w * np.sign(r)) + 0.1 * x


def nan_first(x):
    return float("nan"), np.zeros_like(x)


class NanAt:
    """rosenbrock, but evaluation number k (1-based) returns NaN: k = 3 falls inside the first line search"""

    def __init__(self, k):
        self.k, self.count = k, 0

    def __call__(self, x):
        self.count += 1
        f, g = rosenbrock(x)
        return (float("nan"), g) if self.count == self.k else (f, g)


X_ROSEN = np.array([-1.2, 1.0, -0.5, 0.8, 1.3])
X_QUAD = np.array([3.0, -2.0, 0.5, 1.0, 4.0, -1.5])
X_ABS = np.array([2.0, -1.0, 0.3, 1.7])

# name -> (function factory, x0, parameter overrides of default_lbfgs_params)
LBFGS_CASES = {
    "quadratic": (lambda: quadratic, X_QUAD, {}),
    "rosenbrock": (lambda: rosenbrock, X_ROSEN, {}),
    "abs_restarts": (lambda: abs_sum, X_ABS, dict(past=0)),
    "nan_first": (lambda: nan_first, X_QUAD, {}),
    "nan_in_line_search": (lambda: NanAt(3), X_ROSEN, {}),
    "max_iterations": (lambda: rosenbrock, X_ROSEN, dict(max_iterations=4)),
    "past_delta": (lambda: rosenbrock, X_ROSEN, dict(past=2, delta=1e-2)),
    "g_epsilon_at_start": (lambda: quadratic, X_QUAD, dict(g_epsilon=1e6)),
    "mem_size_1": (lambda: rosenbrock, X_ROSEN, dict(mem_size=1)),
    "max_linesearch": (lambda: rosenbrock, X_ROSEN, dict(max_linesearch=1, nonsmooth_restarts=0)),
    "nonsmooth_restarts_0": (lambda: abs_sum, X_ABS, dict(past=0, nonsmooth_restarts=0)),
}


def run_lbfgs(name):
    make, x0, over = LBFGS_CASES[name]
    fun = make()
    trace = []

    def rec(x):
        trace.append(np.array(x, dtype=np.float64))
        return fun(x)

    rc, x, st = api.lbfgs_minimize(rec, x0, api.default_lbfgs_params(**over))
    tr = np.stack(trace) if trace else np.zeros((0, x0.size))
    return dict(trace=tr, x=x, status=np.int64(rc), final_cost=np.float64(st["final_cost"]), iterations=np.int64(st["iterations"]),
                evaluations=np.int64(st["evaluations"]))


def minco_inputs(N):
    rng = np.random.Generator(np.random.MT19937(1000 + N))
    init_s = rng.normal(0, 1, (3, 3))
    final_s = rng.normal(0, 1, (3, 3))
    final_s[:, 0] += [2.0 * N, 1.0, 0.5]
    q = np.linspace(init_s[:, 0], final_s[:, 0], N + 1)[1:-1].T + rng.normal(0, 0.3, (3, N - 1))
    T = rng.uniform(0.2, 3.0, N)
    gdC = rng.normal(0, 1, (6 * N, 3))
    gdT = rng.normal(0, 1, N)
    return init_s, final_s, q, T, gdC, gdT


def run_minco(N):
    init_s, final_s, q, T, gdC, gdT = minco_inputs(N)
    b, e, gc, gt = api.minco_forward(init_s, final_s, q, T)
    gq, gT = api.minco_propagate(init_s, final_s, q, T, gdC, gdT)
    return dict(coeffs=b, energy=np.float64(e), gradC=gc, gradT=gt, prop_q=gq, prop_T=gT)


def run_mid(cname, N):
    cfg = api.mid_default_config(**mk.CONFIGS[cname])
    init_s, final_s, Q, rots, _ = mk.problem(N, 100 + N)
    rc, x, T, co, fc, it = api.mid_get_ori_traj(init_s, final_s, Q, np.ones(N), rots, cfg)
    return dict(rc=np.int64(rc), x=x, T=T, coeffs=co, cost=np.float64(fc), iterations=np.int64(it))


def main():
    out = {}
    for name in LBFGS_CASES:
        r = run_lbfgs(name)
        print(f"lbfgs {name}: status {int(r['status'])} evaluations {int(r['evaluations'])} iterations {int(r['iterations'])}")
        out.update({f"lbfgs_{name}_{k}": v for k, v in r.items()})
    for N in MINCO_N:
        out.update({f"minco_N{N}_{k}": v for k, v in run_minco(N).items()})
    for cname in mk.CONFIGS:
        for N in MID_N:
            out.update({f"mid_{cname}_N{N}_{k}": v for k, v in run_mid(cname, N).items()})
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
