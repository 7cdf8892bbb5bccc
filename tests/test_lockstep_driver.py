"""CPU: the round driver of the lock-step back end (csrc/host/lockstep.hpp).  tests/cpp/lockstep_driver_main.cpp runs n seeded L-BFGS
minimisations (smooth and kinked functions, some stopped by max_iterations) through the driver svsdf_optimize_lockstep uses, with a CPU
batched evaluator in place of its device round; it is compiled on first use into a temporary directory."""
import os
import shutil
import subprocess
import tempfile

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
HOST = os.path.join(HERE, "..", "implicit_svsdf_planner_b200", "csrc", "host")


@pytest.fixture(scope="module")
def driver():
    d = tempfile.mkdtemp(prefix="lockstep_driver_")
    exe = os.path.join(d, "lockstep_driver_main")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fopenmp", "-ffp-contract=off", "-I", HOST,
                           os.path.join(HERE, "cpp", "lockstep_driver_main.cpp"), "-o", exe])
    yield exe
    shutil.rmtree(d, True)


def run(exe, *args):
    out = subprocess.run([exe, *map(str, args)], capture_output=True, text=True, check=True, timeout=120).stdout.splitlines()
    problems = [ln for ln in out if ln.startswith("P ")]
    s = [ln for ln in out if ln.startswith("S ")][0].split()
    return problems, int(s[1]), int(s[2])


@pytest.mark.parametrize("n,seed", [(1, 1), (5, 2), (40, 3), (97, 4)])
def test_driver_equals_alone(driver, n, seed):
    alone, _, _ = run(driver, "alone", n, seed)
    evals = [int(ln.split()[4]) for ln in alone]
    iters = {int(ln.split()[3]) for ln in alone}
    assert len(iters) > 1 or n == 1  # the problems take different numbers of iterations
    for m in sorted({1, 2, 7, n}):
        got, rounds, violations = run(driver, "lockstep", n, seed, m)
        assert got == alone, f"max_in_flight {m}: iterates differ from the problems minimised alone"
        assert violations == 0, f"max_in_flight {m}: a round fired while a live problem was missing"
        if m == n:
            assert rounds == max(evals)
        else:
            assert rounds >= max(evals)
