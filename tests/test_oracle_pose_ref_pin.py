"""CPU: the pose-sampled obstacle penalty's sample records pinned to the REFERENCE'S OWN grad_cost_p (back_end_optimizer.hpp:956-1028,
cut verbatim into oracle/_ref/libref_pose_portable.so by oracle/ref_extract_pose.py and oracle/ref_pose_shim.cpp).  Where that library
was built the reference runs live and must reproduce tests/golden/ref_pin_pose.npz; everywhere, the oracle's restatement
(oracle/pose_oracle.py), which the GPU tests check the kernel against, must equal the golden bit for bit: every analytic shape and the
Polygon, with and without poly_params, on the star map and a five-layer map, with poses outside the map, boxes clipped at every
face, yaws selecting one, all or no layers, voxels exactly at |p_rel| = half, and the four smoothed-L1 regimes."""
import os

import numpy as np
import pytest

from oracle import k3_points, pose_oracle, ref_pose_py

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pin_pose.npz")


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.uint64)


def load():
    g = np.load(GOLD)
    maps = {}
    for mi in range(2):
        occ = g[f"map{mi}_occ"].astype(bool)
        lo = g[f"map{mi}_lo"]
        res = float(g[f"map{mi}_res"])
        gm = k3_points.GridMap3D(lo, lo + np.array(occ.shape) * res, res, occ)
        maps[mi] = (gm, tuple(g[f"map{mi}_half"]))
    cases = [(k, int(g["case_map"][k]), str(g["case_shape"][k]), tuple(g["case_pp"][k]), g[f"case{k}_poses"], g[f"case{k}_rec"])
             for k in range(len(g["case_map"]))]
    return g, maps, cases


G, MAPS, CASES = load()


@pytest.mark.parametrize("k", range(len(CASES)))
def test_oracle_is_the_reference(k):
    _, mi, shape, pp, poses, rec = CASES[k]
    gm, half = MAPS[mi]
    got = np.array([pose_oracle.grad_cost_p(gm, shape, p, half, float(G["safety_hor"]), pp) for p in poses])
    assert np.array_equal(bits(got), bits(rec)), (shape, pp, np.argwhere(bits(got) != bits(rec))[:5])


@pytest.mark.skipif(not ref_pose_py.available("portable"), reason="the reference pin is built only where the reference tree is")
@pytest.mark.parametrize("k", range(0, len(CASES), 7))
def test_live_reference_reproduces_the_golden(k):
    _, mi, shape, pp, poses, rec = CASES[k]
    gm, half = MAPS[mi]
    live = ref_pose_py.grad_cost_p(shape, pp, gm.occ, gm.boundary_min, gm.res, half, float(G["safety_hor"]), poses)
    assert np.array_equal(bits(live), bits(rec))


def test_the_golden_reaches_its_edges():
    """The golden holds what it claims: every shape with and without poly_params on both maps, active and inactive samples, poses
    outside the map, voxels kept at |p_rel| = half on each axis, and the cubic part of smoothed L1."""
    assert len({(c[1], c[2], c[3]) for c in CASES}) == 72
    gm, half = MAPS[1]
    kept_at_half = 0
    cubic = 0
    for _, mi, shape, pp, poses, rec in CASES:
        assert (rec[:, 0] > 0).any() and (rec[:, 0] == 0).any(), (mi, shape, pp)
        if mi != 1 or shape != "Circle" or pp != (0.0, 0.0, 0.0):
            continue
        for p, r in zip(poses, rec):
            _, kept, active = pose_oracle.grad_cost_p(gm, shape, p, half, 0.7, pp, with_cells=True)
            if (11, 11, 2) in kept and any(abs(abs(v) - h) == 0.0 for v, h in zip((6.5 - p[0], -0.5 - p[1], 0.0 - p[2]), half)):
                kept_at_half += 1
        cubic = int(np.sum((rec[-4:, 0] > 0) & (rec[-4:, 0] < 0.01)))  # the regime poses come last
    assert kept_at_half >= 6
    assert cubic >= 1
