"""CPU: oracle/clearance_oracle.py, the dense restatement of svsdf_map_clearance that the GPU tests check against — values at known
distances from a Circle robot's straight path (outside and on the path), the list order and its summary (ties, an empty list,
d_max = 0), and 3-D columns (stacked voxels count once, a voxel above layer 0 counts)."""
import math

import numpy as np
import pytest

from oracle import clearance_oracle as co


def line_traj(L=6.0, dur=3.0, yaw=0.0):
    """A single piece: straight along x from (0, 0) to (L, 0) at constant yaw."""
    b = np.zeros((6, 3))
    b[0, 2] = yaw
    b[1, 0] = L / dur
    return np.array([dur]), b.T.reshape(-1).copy()


def test_circle_on_a_line_known_distances(oracle_mod):
    orc = oracle_mod.Oracle("Circle")  # radius 1
    T, c = line_traj()
    orc.set_traj(T, c)
    res, origin = 0.5, (-5.0, -5.0)  # centre of cell (i, j): ((i + 0.5) 0.5 - 5, (j + 0.5) 0.5 - 5)
    occ = np.zeros((30, 30), dtype=bool)
    cells = {(16, 14): 2.25, (16, 16): 3.25, (16, 4): 2.75, (25, 10): None, (16, 9): 0.25, (12, 10): 0.25}
    for ij in cells:
        occ[ij] = True
    r = co.clearance(orc, occ, origin, res)
    assert [tuple(x) for x in r["ij"]] == sorted(cells)  # ascending i * Y + j
    assert r["n_occupied"] == r["n_evaluated"] == r["n_within"] == len(cells)
    assert np.array_equal(r["xy"], (r["ij"] + 0.5) * res + np.array(origin))
    for (ij, d), xy, v in zip(sorted(cells.items()), r["xy"], r["sdf"]):
        if d is None:  # (7.75, 0.25): past the end of the path, distance to the end point (6, 0)
            d = math.hypot(xy[0] - 6.0, xy[1])
        # outside: the outer solve's distance - r; inside: the interior (GSIP) depth -(r - distance), to its ring sampling's precision
        assert abs(v - (d - 1.0)) < (1e-6 if d > 1.0 else 1e-2), (ij, v, d)
    inside = r["sdf"] <= 0.0
    assert r["n_colliding"] == int(inside.sum()) == 2  # the two cells 0.25 from the path
    assert r["min_sdf"] == r["sdf"][r["argmin"]] < 0.0
    # at d_max = 1.5: only the cells within 2.5 of the path remain, in the same order
    r2 = co.clearance(orc, occ, origin, res, d_max=1.5)
    assert r2["n_within"] == 4 and r2["n_occupied"] == 6
    assert np.array_equal(r2["sdf"], r["sdf"][r["sdf"] <= 1.5])


def test_summary_ties_empty_and_zero():
    ij = np.array([[0, 1], [0, 3], [2, 0], [2, 5], [4, 4]])
    xy = ij + 0.5
    ts = np.arange(5.0)
    r = co.summarise(ij, xy, [0.5, 0.2, 0.9, 0.2, 0.2], ts, 0.7, 5)
    assert r["n_within"] == 4 and r["argmin"] == 1 and r["min_sdf"] == 0.2  # the first of three equal minima
    assert np.array_equal(r["ij"], ij[[0, 1, 3, 4]]) and np.array_equal(r["tstar"], ts[[0, 1, 3, 4]])
    e = co.summarise(ij, xy, [1.0, 2.0, 3.0, 4.0, 5.0], ts, 0.7, 5)
    assert e["n_within"] == 0 and e["min_sdf"] == math.inf and e["argmin"] == -1 and e["n_colliding"] == 0
    z = co.summarise(ij, xy, [0.0, 1e-300, -0.0, -2.0, 3.0], ts, 0.0, 5)  # d_max = 0: a value of exactly 0 is listed and colliding
    assert z["n_within"] == 3 and z["n_colliding"] == 3 and z["argmin"] == 2 and z["min_sdf"] == -2.0
    assert np.array_equal(z["ij"], ij[[0, 2, 3]])
    for bad in (-1e-12, -1.0, float("nan"), -math.inf):
        with pytest.raises(ValueError):
            co.summarise(ij, xy, ts, ts, bad, 5)
    assert co.summarise(ij, xy, ts, ts, math.inf, 5)["n_within"] == 5


def test_three_d_columns():
    occ = np.zeros((4, 5, 3), dtype=bool)
    occ[1, 2, 0] = occ[1, 2, 1] = occ[1, 2, 2] = True  # stacked: one column
    occ[3, 0, 2] = True                                # only above layer 0
    occ[0, 4, 1] = True
    ij = co.occupied_columns(occ)
    assert [tuple(x) for x in ij] == [(0, 4), (1, 2), (3, 0)]
    assert np.array_equal(co.occupied_columns(occ[:, :, 0]), [[1, 2]])
    assert co.centres(ij, (0.1, -0.2), 0.3).tolist() == [[(0 + 0.5) * 0.3 + 0.1, (4 + 0.5) * 0.3 - 0.2],
                                                          [(1 + 0.5) * 0.3 + 0.1, (2 + 0.5) * 0.3 - 0.2],
                                                          [(3 + 0.5) * 0.3 + 0.1, (0 + 0.5) * 0.3 - 0.2]]


def test_empty_map_and_three_d_oracle(oracle_mod):
    orc = oracle_mod.Oracle("Circle")
    T, c = line_traj()
    orc.set_traj(T, c)
    r = co.clearance(orc, np.zeros((8, 8, 2), dtype=bool), (0.0, 0.0), 1.0)
    assert r["n_occupied"] == r["n_within"] == 0 and r["argmin"] == -1 and r["min_sdf"] == math.inf
    occ = np.zeros((8, 8, 3), dtype=bool)
    occ[3, 0, 0] = occ[3, 0, 1] = True  # centre (2.5, -0.5): 0.5 from the path
    occ[5, 4, 2] = True                 # centre (4.5, 3.5): 3.5 from the path
    r = co.clearance(orc, occ, (-1.0, -1.0), 1.0)
    assert r["n_occupied"] == 2 and r["n_colliding"] == 1
    assert abs(r["sdf"][0] + 0.5) < 1e-2 and abs(r["sdf"][1] - 2.5) < 1e-6
