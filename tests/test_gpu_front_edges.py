"""The A* front end on the GPU at the limits of its inputs, bit for bit against the reference's own code and the oracle.

Entry points: front_init / front_kernels (initShape), front_cspace (k_cspace: kernelConv over every yaw kernel and cell),
front_check_kernel_value, front_expand (ok, child yaw, parts mask: k_expand_nodes / node_test), front_astar and
front_astar_device (paths, expansions, status).  The case matrix is tests/front_cases.py (every shape with and without a
pre-transform; resolutions 0.1, 0.25, 1 and 2.5 at origin (-12.37, 3.1); half boxes from 0.4 to 160 cells per side, so the
32-cells-per-ballot loop runs from one to hundreds of rounds; X or Y = 1; Y = 0, 1, 31 mod 32; empty and full maps; yaw
counts 1 to 64; father yaws at -pi, its neighbouring doubles, the kernel boundaries and outside [-pi, pi)).  front_cspace is
also read as the raw words of the C ABI, so that the bits past Y (which must read 0) are seen.

Where the reference's code is defined the device is held to tests/golden/ref_pin_front.npz (the reference's outputs); on every
node of every case, including the Circle, the initShape overruns (K = 3, 36, 63) and father yaws whose index must be clamped,
it is held to the oracle (tests/test_oracle_front_ref_pin.py ties the oracle to the reference).
"""
import ctypes as C
import os

import numpy as np
import pytest

import front_cases as FC
from implicit_svsdf_planner_b200 import api, batch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pin_front.npz")


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN, allow_pickle=False) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="module")
def oracle_all(oracle_mod):
    return FC.oracle_records(oracle_mod, all_nodes=True)


def _ctx(c, occ):
    ctx = api.Context(c["shape"], poly_params=c["pp"])
    ctx.front_init(c["ks"], c["K"], c["res"], c["safeh"])
    ctx.set_map(batch.pack_map_kernel(occ, c["ks"]), c["X"], c["Y"], c["ks"], FC.ORIGIN, c["res"])
    return ctx


def _raw_cspace(ctx, c):
    """svsdf_front_cspace's words [K, X, ceil(Y / 32)] as the C ABI returns them, padding bits included."""
    W = (c["Y"] + 31) // 32
    words = np.full((c["K"], c["X"], W), 0xFFFFFFFF, dtype=np.uint32)  # anything the kernel leaves unwritten shows up
    ms = C.c_float()
    rc = api.lib().svsdf_front_cspace(ctx.h, words.ctypes.data_as(C.c_void_p), C.byref(ms), None)
    assert rc == 0, rc
    return words


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize("i", range(2 * len(FC.SHAPES)))
def test_node_test_at_the_edges(golden, oracle_all, i):
    c = FC.expand_cases()[i]
    occ, ij, fy = FC.expand_inputs(c)
    ctx = _ctx(c, occ)
    _, _, byt = ctx.front_kernels()
    free, _ = ctx.front_cspace(c["X"], c["Y"])
    words = _raw_cspace(ctx, c)
    ok, cy, parts = ctx.front_expand(ij, fy)
    ok1, cy1 = ctx.front_check_kernel_value(fy, ij)
    ctx.close()
    got = {"kern": FC.digest(byt), "cspace": FC.digest(free)}
    # the C ABI's words: cells beyond Y read 0 (not free), and the first Y bits are the map above
    bits = np.unpackbits(words.byteswap().view(np.uint8).reshape(c["K"], c["X"], -1), axis=2)
    assert not bits[:, :, c["Y"]:].any(), (i, c["Y"])
    assert np.array_equal(bits[:, :, : c["Y"]].astype(bool), free), i
    # the oracle, on every node
    for f in ("kern", "cspace"):
        assert got[f] == str(oracle_all[f"e{i}_{f}"]), (i, f)
    assert np.array_equal(ok, oracle_all[f"e{i}_ok"].astype(bool)), i
    assert np.array_equal(parts, oracle_all[f"e{i}_parts"]), (i, np.argwhere(parts != oracle_all[f"e{i}_parts"])[:5].tolist())
    assert np.array_equal(_bits(cy), _bits(oracle_all[f"e{i}_cy"])), i
    assert np.array_equal(ok1, oracle_all[f"e{i}_ckv_ok"].astype(bool)), i
    assert np.array_equal(_bits(cy1[ok1]), _bits(oracle_all[f"e{i}_ckv_cy"][ok1])), i
    # the reference's own outputs, where its code is defined
    if f"e{i}_ok" not in golden:
        return
    d = FC.ref_defined(c, fy)
    assert FC.digest(batch.pack_map_kernel(occ, c["ks"])) == str(golden[f"e{i}_mk"])
    for f in ("kern", "cspace"):
        assert got[f] == str(golden[f"e{i}_{f}"]), (i, f)
    assert np.array_equal(ok[d], golden[f"e{i}_ok"].astype(bool)) and np.array_equal(parts[d], golden[f"e{i}_parts"]), i
    assert np.array_equal(_bits(cy[d]), _bits(golden[f"e{i}_cy"])), i
    g_ok = golden[f"e{i}_ckv_ok"].astype(bool)
    assert np.array_equal(ok1[d], g_ok) and np.array_equal(_bits(cy1[d][g_ok]), _bits(golden[f"e{i}_ckv_cy"][g_ok])), i


@pytest.mark.parametrize("i", range(2 * len(FC.SHAPES)))
def test_searches_at_the_edges(golden, oracle_all, i):
    c = FC.search_cases()[i]
    occ, st, go = FC.search_inputs(c)
    ctx = _ctx(c, occ)
    paths_d, ex_d, status, _ = ctx.front_astar_device(st, go, max_path=4096)
    paths_h, ex_h, _ = ctx.front_astar(st, go, max_path=4096)
    ctx.close()
    for paths, ex in ((paths_d, ex_d), (paths_h, ex_h)):
        lens, cat = FC.pack_paths(paths)
        for want in (oracle_all, golden) if f"s{i}_len" in golden else (oracle_all,):
            assert np.array_equal(lens, want[f"s{i}_len"]) and np.array_equal(ex, want[f"s{i}_ex"]), i
            assert np.array_equal(_bits(cat), _bits(want[f"s{i}_path"])), i
    found = oracle_all[f"s{i}_found"].astype(bool)
    assert status[4] == 0  # the start lies outside the map
    assert np.array_equal(status[:4], np.where(found[:4], 1, 2)), (i, status)


@pytest.mark.parametrize("ks,K", [(33, 18), (16, 18), (2, 18), (0, 18), (17, 65), (17, 0)])
def test_refused_sizes(ks, K):
    """Kernel sizes above 32 or even, and yaw counts outside 1..64, are refused before anything is launched."""
    ctx = api.Context("star")
    with pytest.raises(api.SvsdfError):
        ctx.front_init(ks, K, 1.0, 0.0)
    ctx.front_init(31, 64, 1.0, 0.0)  # the largest accepted sizes
    _, cells, _ = ctx.front_kernels()
    assert cells.shape == (64, 31, 31)
    ctx.close()
