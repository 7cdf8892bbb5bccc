"""CPU tests: the host L-BFGS (host/lbfgs.hpp, a resumable machine on flat storage) and MINCO (host/minco.hpp, SVSDF_HD functions on
flat storage) give the bits they gave before that restatement, which the device back end (svsdf_optimize_device) shares.  Golden
outputs: tests/golden/host_backend.npz (tests/golden/make_backend_golden.py)."""
import os
import sys

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_backend_golden as mk  # noqa: E402  (the callbacks, seeded inputs and the calls that recorded the golden outputs)


@pytest.fixture(scope="module")
def gold():
    return np.load(mk.OUT)


def same_bits(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


@pytest.mark.parametrize("name", list(mk.LBFGS_CASES))
def test_lbfgs_iterates_and_exit_are_unchanged(gold, name):
    """Every evaluated x in order, the returned x, status, cost, iterations and evaluations, on one callback per exit of the solver."""
    r = mk.run_lbfgs(name)
    k = f"lbfgs_{name}_"
    assert same_bits(r["trace"], gold[k + "trace"])
    assert same_bits(r["x"], gold[k + "x"])
    for f in ("status", "iterations", "evaluations"):
        assert int(r[f]) == int(gold[k + f]), f
    assert same_bits(r["final_cost"], gold[k + "final_cost"])


def test_lbfgs_cases_reach_their_exits(gold):
    """The callbacks do reach the exits they are named for."""
    st = {name: int(gold[f"lbfgs_{name}_status"]) for name in mk.LBFGS_CASES}
    assert st["abs_restarts"] == 3 and st["nan_first"] == st["nan_in_line_search"] == -1012
    assert st["max_iterations"] == -1008 and st["past_delta"] == 1 and st["g_epsilon_at_start"] == 0
    assert st["max_linesearch"] == st["nonsmooth_restarts_0"] == -1009
    assert int(gold["lbfgs_g_epsilon_at_start_evaluations"]) == 1


@pytest.mark.parametrize("N", mk.MINCO_N)
def test_minco_forward_and_propagate_are_unchanged(gold, N):
    r = mk.run_minco(N)
    for f, v in r.items():
        assert same_bits(v, gold[f"minco_N{N}_{f}"]), f


@pytest.mark.parametrize("cname", list(mk.mk.CONFIGS))
@pytest.mark.parametrize("N", mk.MID_N)
def test_mid_end_reference_patch_mode_is_unchanged(gold, cname, N):
    """svsdf_mid_get_ori_traj runs the L-BFGS in its reference_patch mode (Armijo-only, steepest-descent fallback evaluations)."""
    r = mk.run_mid(cname, N)
    for f, v in r.items():
        assert same_bits(v, gold[f"mid_{cname}_N{N}_{f}"]), f
