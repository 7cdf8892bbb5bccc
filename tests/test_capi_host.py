"""CPU: the C-ABI shared library loads, exports every symbol include/svsdf.h declares, its host-only entry points
(MINCO, tau maps, L-BFGS, registry) agree with the oracle, and it refuses to run the hot path without a GPU (no
CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
from conftest import HAS_GPU  # noqa: E402


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "svsdf.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = sorted(set(re.findall(r"\b(svsdf_[a-z0-9_A-Z]+)\s*\(", hdr)))
    declared = [d for d in declared if not d.endswith("_t")]
    assert len(declared) >= 25
    L = api.lib()
    for name in declared:
        assert hasattr(L, name), f"{name} declared in include/svsdf.h but not exported"
    assert sorted(api.EXPORTED_SYMBOLS) == declared


def test_library_is_built_for_sm90a_only():
    out = os.popen(f"cuobjdump -lelf {api.LIB_PATH} 2>/dev/null").read()
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_shape_registry_matches_reference_keys():
    L = api.lib()
    names = ["star", "sdHorseshoe", "sdPie", "sdPie2", "sdArc", "sdTunnel", "sdCutDisk", "sdTrapezoid", "sdRhombus",
             "sdHeart", "sdRoundedX", "bigX", "sdRoundedCross", "sdOrientedVesica", "sdMoon", "sdUnevenCapsule"]
    assert [L.svsdf_shape_id(n.encode()) for n in names] == list(range(16))
    assert L.svsdf_shape_id(b"unknown_mesh") == 17 and L.svsdf_shape_id(None) == 17


@pytest.mark.parametrize("N", [2, 5, 8, 16, 40])
def test_host_minco_matches_oracle(oracle_mod, N):
    init_s, final_s, q, T = scenes.make_trajectory("star", N, 100 + N)
    rng = np.random.default_rng(N)
    T = T * rng.uniform(0.5, 1.8, size=N)
    init_s[:, 1] = rng.normal(size=3)
    final_s[:, 2] = rng.normal(size=3)
    b0, e0, gc0, gt0 = oracle_mod.minco_forward(init_s, final_s, q, T)
    b1, e1, gc1, gt1 = api.minco_forward(init_s, final_s, q, T)
    scale = max(1.0, np.abs(b0).max())
    assert np.abs(b1 - b0).max() <= 1e-11 * scale
    assert abs(e1 - e0) <= 1e-11 * abs(e0)
    assert np.abs(gc1 - gc0).max() <= 1e-11 * max(1.0, np.abs(gc0).max())
    assert np.abs(gt1 - gt0).max() <= 1e-11 * max(1.0, np.abs(gt0).max())
    W = rng.normal(size=(6 * N, 3))
    wT = rng.normal(size=N)
    gq0, gT0 = oracle_mod.minco_propagate(init_s, final_s, q, T, gc0 + W, gt0 + wT)
    gq1, gT1 = api.minco_propagate(init_s, final_s, q, T, gc0 + W, gt0 + wT)
    assert np.abs(gq1 - gq0).max() <= 1e-10 * max(1.0, np.abs(gq0).max())
    assert np.abs(gT1 - gT0).max() <= 1e-10 * max(1.0, np.abs(gT0).max())


def test_tau_maps_match_reference_formulas():
    T = np.array([0.05, 0.5, 1.0, 1.0000001, 2.5, 100.0])
    tau = api.backward_T(T)
    assert np.abs(api.forward_T(tau) - T).max() < 1e-10
    assert np.array_equal(tau, scenes.backward_T(T))
    assert np.array_equal(api.forward_T(tau), scenes.forward_T(tau))


def test_host_lbfgs_follows_lbfgs_ref(oracle_mod):
    """Same algorithm as the oracle's restatement of lbfgs_ref.hpp -> same iterates on a smooth and a nonsmooth test."""
    L = oracle_mod.lib()
    CB = C.CFUNCTYPE(C.c_double, C.c_void_p, oracle_mod.dp, oracle_mod.dp, C.c_int)
    L.orc_lbfgs_cb.argtypes = [CB, C.c_void_p, oracle_mod.dp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, oracle_mod.dp]

    def rosen10(x):
        f = np.sum(100.0 * (x[1:] - x[:-1] ** 2) ** 2 + (1 - x[:-1]) ** 2)
        g = np.zeros_like(x)
        g[:-1] += -400 * x[:-1] * (x[1:] - x[:-1] ** 2) - 2 * (1 - x[:-1])
        g[1:] += 200 * (x[1:] - x[:-1] ** 2)
        return f, g

    def nonsmooth(x):  # piecewise smooth: |x0| + 2|x1 - 1| + (x2 + 3)^2
        f = abs(x[0]) + 2 * abs(x[1] - 1) + (x[2] + 3) ** 2
        return f, np.array([np.sign(x[0]), 2 * np.sign(x[1] - 1), 2 * (x[2] + 3)])

    for fun, x0, past, delta, geps in ((rosen10, np.full(10, -1.2), 0, 1e-6, 1e-8), (nonsmooth, np.array([3.0, -2.0, 5.0]), 3, 1e-9, 0.0)):
        def cbf(_i, xp, gp, n):
            f, g = fun(np.ctypeslib.as_array(xp, shape=(n,)).copy())
            np.ctypeslib.as_array(gp, shape=(n,))[:] = g
            return float(f)

        cb = CB(cbf)
        xo = x0.copy()
        so = np.zeros(3)
        ro = L.orc_lbfgs_cb(cb, None, xo.ctypes.data_as(oracle_mod.dp), xo.size, 8, past, delta, geps, 200, so.ctypes.data_as(oracle_mod.dp))
        rp, xp_, sp = api.lbfgs_minimize(fun, x0, api.default_lbfgs_params(mem_size=8, past=past, delta=delta, g_epsilon=geps, max_iterations=200))
        assert rp == ro and sp["iterations"] == int(so[1]) and sp["evaluations"] == int(so[2])
        assert np.abs(xp_ - xo).max() < 1e-12
    assert abs(sp["final_cost"]) < 1e-3  # the nonsmooth problem's minimum is 0 at (0, 1, -3)


def test_invalid_arguments_are_rejected_without_gpu():
    L = api.lib()
    h = C.c_void_p()
    assert L.svsdf_create(None, C.byref(h)) == -1
    assert L.svsdf_minco_forward(None, None, 8, None, None, None, None, None, None) == -1
    assert L.svsdf_set_points(None, None, 0, 3) == -1


@pytest.mark.skipif(HAS_GPU, reason="checks the behaviour on a machine without a CUDA device")
def test_no_cpu_fallback_without_gpu():
    with pytest.raises(api.SvsdfError):
        api.Context("star")


def test_product_never_touches_the_oracle():
    pkg = os.path.join(ROOT, "implicit_svsdf_planner_b200")
    offenders = []
    for dp_, _, files in os.walk(pkg):
        if os.sep + "lib" in dp_:
            continue
        for f in files:
            if f.endswith((".py", ".cpp", ".cu", ".cuh", ".h", ".hpp")):
                txt = open(os.path.join(dp_, f), errors="ignore").read()
                if re.search(r"(from|import)\s+oracle|oracle_py|#include\s+\"[^\"]*oracle|libsvsdf_oracle", txt):
                    offenders.append(os.path.join(dp_, f))
    assert not offenders, offenders


def test_lbfgs_nonsmooth_restarts_and_failed_first_evaluation():
    """(i) On a cost with kinks the plain Lewis-Overton L-BFGS ends with a negative line-search code; with
    nonsmooth_restarts it drops the quasi-Newton memory at the kink, continues along -g and ends with a non-negative status
    (3 = no more progress at a kink) at a point at least as good.  (ii) A first evaluation that returns NaN is an error of
    the run (LBFGSERR_INVALID_FUNCVAL = -1012), never 'convergence' (ADVICE r1)."""
    from implicit_svsdf_planner_b200 import api

    def fun(x):  # |x0| + |x1| with a subgradient that is wrong left of the kink: no step satisfies Armijo + weak Wolfe
        return float(np.abs(x).sum()), np.ones_like(x)

    x0 = np.array([1.0, 2.0])
    p0 = api.default_lbfgs_params(mem_size=8, past=0, delta=0.0, g_epsilon=1e-9, max_iterations=50)
    p0.nonsmooth_restarts = 0
    rc0, xa, st0 = api.lbfgs_minimize(fun, x0, p0)
    p1 = api.default_lbfgs_params(mem_size=8, past=0, delta=0.0, g_epsilon=1e-9, max_iterations=50)
    assert p1.nonsmooth_restarts == 8  # library default
    rc1, xb, st1 = api.lbfgs_minimize(fun, x0, p1)
    assert rc0 in (-1009, -1011, -1007) and rc1 == 3, (rc0, rc1)
    assert st1["final_cost"] <= st0["final_cost"] + 1e-12
    assert abs(fun(xb)[0] - st1["final_cost"]) < 1e-12  # the reported cost is the cost of the returned iterate

    rcn, _, _ = api.lbfgs_minimize(lambda x: (float("nan"), np.zeros_like(x)), x0, p1)
    assert rcn == -1012


def test_lmbm_plugin_equals_the_library_and_private_copies_run_concurrently(tmp_path):
    """svsdf_lmbm_open / svsdf_lmbm_minimize on the host (no GPU): same result as calling the library's lmbm_optimize directly, and two
    private copies minimise concurrently from two threads (LMBM keeps its callback and its state in statics — one shared instance
    cannot).  The library is tests/cpp/lmbm_standin.cpp: LMBM's entry point with its callback in statics (the reference's binary is
    not redistributed).  Runs in a subprocess (tests/tools/lmbm_plugin_check.py)."""
    import json
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    so = str(tmp_path / "liblmbm_standin.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", os.path.join(root, "tests", "cpp", "lmbm_standin.cpp"), "-o", so])
    out = subprocess.run([sys.executable, os.path.join(root, "tests", "tools", "lmbm_plugin_check.py"), "--lib", so], capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    rec = json.loads(out.stdout.strip().split("\n")[-1])
    assert rec["direct_equal"] and rec["concurrent_equal_alone"] and rec["status"] >= 0 and rec["f"] < 0.1 * rec["f_start"]
    # a wrong path is an error with a message, not a crash
    from implicit_svsdf_planner_b200 import api

    with pytest.raises(api.SvsdfError):
        api.Lmbm(os.path.join(root, "no_such_lmbm.so"))
