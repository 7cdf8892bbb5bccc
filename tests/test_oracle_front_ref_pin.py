"""The A* front end of the oracle (oracle/frontend_oracle.hpp) against the reference's OWN code, bit for bit.

The reference side is kernelConv / visit_kernels_by_distance / checkKernelValue / checkSubSWCollision (sw_manager.hpp),
getPointsInAABB2D / projInMap (PCSmap_manager.h), the GridMap3D index and centre helpers, and AstarGetSucc /
AstarPathSearch / getPath (front_end_Astar.hpp), cut verbatim and compiled by `make -C oracle ref` (portable sin/cos).  It runs
live where oracle/_ref/libref_front_portable.so exists, and is read from tests/golden/ref_pin_front.npz otherwise.  The case
matrix is tests/front_cases.py: every shape with and without a pre-transform, resolutions 0.1 to 2.5, half boxes from under one
cell to 160 cells, edge and corner nodes, the edges of the father-yaw index, and a search scene per shape.
"""
import os

import numpy as np
import pytest

import front_cases as FC
from oracle import ref_front_py

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pin_front.npz")


@pytest.fixture(scope="module")
def reference():
    if ref_front_py.available("portable"):
        return FC.reference_records("portable"), "live"
    with np.load(GOLDEN, allow_pickle=False) as z:
        return {k: z[k] for k in z.files}, "fixture"


@pytest.fixture(scope="module")
def oracle_rec(oracle_mod):
    return FC.oracle_records(oracle_mod)


def test_fixture_matches_live_reference(reference):
    rec, src = reference
    if src != "live":
        pytest.skip("the reference's front end is not built here; the other tests read the fixture")
    with np.load(GOLDEN, allow_pickle=False) as z:
        assert sorted(z.files) == sorted(rec)
        for k in z.files:
            assert np.array_equal(z[k], rec[k]), k


def test_matrix_reaches_its_edges(reference):
    rec, _ = reference
    parts = np.concatenate([rec[k].ravel() for k in rec if k.endswith("_parts")])
    assert set(np.unique(parts).tolist()) >= {0, 1, 2, 3, 4, 6, 7}  # the three conditions pass and fail in most combinations
    cases = FC.expand_cases()
    assert sum(f"e{i}_ok" in rec for i in range(len(cases))) >= 20
    found = np.concatenate([rec[k] for k in rec if k.endswith("_found")])
    assert found.sum() >= 15 and (found == 0).sum() >= 15
    # the half box spans < 1 cell and > 100 cells per side; a yaw right at -pi and one a double below the kernel boundary are pinned
    hb_cells = [(c["ks"] // 2 + 1) / c["res"] for c in cases]
    assert min(hb_cells) < 1 and max(hb_cells) > 100
    assert -FC.PI_CODE in FC.father_yaws(18)
    # father yaws whose index the product clamps (the reference's is undefined there): compared with the oracle on the GPU
    clamped = 0
    for c in cases:
        fi = FC.father_index(c["K"], FC.expand_inputs(c)[2])
        clamped += int(((fi < 0) | (fi >= c["K"])).sum())
    assert clamped >= 100


@pytest.mark.parametrize("i", range(2 * len(FC.SHAPES)))
def test_node_test_is_the_references(reference, oracle_rec, i):
    rec, _ = reference
    if f"e{i}_ok" not in rec:
        pytest.skip("case outside the reference's defined inputs (Circle, or an initShape yaw loop that overruns)")
    for f in ("kern", "cspace", "aabb", "ok", "parts", "ckv_ok"):
        assert np.array_equal(oracle_rec[f"e{i}_{f}"], rec[f"e{i}_{f}"]), (i, f)
    for f in ("cy", "ckv_cy"):  # bit for bit
        assert np.array_equal(oracle_rec[f"e{i}_{f}"].view(np.uint64), rec[f"e{i}_{f}"].view(np.uint64)), (i, f)


@pytest.mark.parametrize("i", range(2 * len(FC.SHAPES)))
def test_search_is_the_references(reference, oracle_rec, i):
    rec, _ = reference
    if f"s{i}_len" not in rec:
        pytest.skip("the reference's Circle has no kernels")
    for f in ("len", "ex", "found"):
        assert np.array_equal(oracle_rec[f"s{i}_{f}"], rec[f"s{i}_{f}"]), (i, f)
    assert np.array_equal(oracle_rec[f"s{i}_path"].view(np.uint64), rec[f"s{i}_path"].view(np.uint64)), i


def test_glibc_variant_gives_the_same_booleans_and_paths():
    """The reference as it runs (glibc sin/cos) against the pinned portable build: every record agrees on this matrix (DESIGN.md §4
    has a denser scene where they do not)."""
    if not ref_front_py.available("glibc"):
        pytest.skip("the reference's front end is not built here")
    a, b = FC.reference_records("portable"), FC.reference_records("glibc")
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(a[k], b[k]), k
