"""The LMBM plug-in on top of the GPU callback: a library exporting lmbm::lmbm_optimize (lmbm.h:214-221) minimises `svsdf_evaluate` —
the drop-in of INTEGRATION.md §2 — once handed the C entry point from outside and once loaded by the context itself
(svsdf_set_lmbm_library + svsdf_optimize).  The library is tests/cpp/lmbm_standin.cpp, which has LMBM's entry point and keeps its
callback in statics like LMBM does (the reference's prebuilt binary is not redistributed); the reference's own LMBM run is replayed
through svsdf_evaluate by tests/test_gpu_parity.py::test_replay_of_the_reference_lmbm_trace."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def run(args):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "tools", "run_lmbm_gpu.py")] + args, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    return json.loads(out.stdout.strip().split("\n")[-1])


def test_lmbm_as_the_contexts_own_solver_plugin(tmp_path):
    """svsdf_set_lmbm_library: the context loads a private instance of the library and svsdf_optimize runs it on svsdf_evaluate — the
    same run, bit for bit, as handing the entry point to lmbm_optimize from outside."""
    so = str(tmp_path / "liblmbm_standin.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", os.path.join(ROOT, "tests", "cpp", "lmbm_standin.cpp"), "-o", so])
    direct = run(["--lib", so])
    plug = run(["--lib", so, "--plugin"])
    assert int(plug["lmbm_return"]) == int(direct["lmbm_return"]) and plug["f_final"] == direct["f_final"]
    assert plug["iterations"] == direct["iterations"]
    assert plug["optimize_return"] == (1 if plug["lmbm_return"] == 0 else plug["lmbm_return"])  # 0 remapped to 1, back_end_optimizer.cpp:66-69
    assert plug["f_final"] < 0.6 * plug["f_start"]
