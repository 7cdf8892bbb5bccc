"""CPU: plan.new_cells, the repair rule (which listed cells a clearance adds to the query set), on hand-made inputs, and the bookkeeping
of plan.Repair on a hand-made sequence of certificates."""
import math

import numpy as np

from implicit_svsdf_planner_b200 import api, plan


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.uint64)


def test_bit_equal_duplicates_dropped_one_ulp_kept():
    q = np.array([[0.1, 0.2], [1.5, -2.25]])
    cells = np.array([[0.1, 0.2], [np.nextafter(0.1, 1.0), 0.2], [1.5, np.nextafter(-2.25, 0.0)], [1.5, -2.25]])
    out = plan.new_cells(cells, q)
    assert np.array_equal(bits(out), bits(cells[1:3]))


def test_signed_zero_is_not_bit_equal():
    out = plan.new_cells(np.array([[-0.0, 1.0], [0.0, 1.0]]), np.array([[0.0, 1.0]]))
    assert np.array_equal(bits(out), bits([[-0.0, 1.0]]))


def test_stacked_query_repeats_count_as_one_column():
    # the extraction lists a column once per z layer (P x 3 here, and P x 2 with repeated rows): any of them makes the column known
    q3 = np.array([[2.0, 3.0, 0.0], [2.0, 3.0, 0.5], [2.0, 3.0, 1.0], [4.0, 5.0, 0.0]])
    cells = np.array([[2.0, 3.0], [4.0, 5.0], [6.0, 7.0]])
    assert np.array_equal(bits(plan.new_cells(cells, q3)), bits([[6.0, 7.0]]))
    assert np.array_equal(bits(plan.new_cells(cells, q3[:, :2])), bits([[6.0, 7.0]]))


def test_list_order_kept_and_each_column_once():
    cells = np.array([[5.0, 1.0], [-3.0, 2.0], [5.0, 1.0], [0.5, 0.5], [-3.0, 2.0]])
    out = plan.new_cells(cells, np.array([[0.5, 0.5]]))
    assert np.array_equal(bits(out), bits([[5.0, 1.0], [-3.0, 2.0]]))


def test_empty_inputs():
    assert plan.new_cells(np.empty((0, 2)), np.array([[1.0, 2.0]])).shape == (0, 2)
    assert plan.new_cells(np.empty((0, 2)), np.empty((0, 2))).shape == (0, 2)
    cells = np.array([[1.0, 2.0]])
    assert np.array_equal(bits(plan.new_cells(cells, np.empty((0, 2)))), bits(cells))


def clearance(xy, sdf):
    xy = np.asarray(xy, dtype=np.float64).reshape(-1, 2)
    sdf = np.asarray(sdf, dtype=np.float64)
    k = int(np.argmin(sdf)) if len(sdf) else -1
    return api.Clearance(0.7, np.zeros((len(xy), 2), dtype=np.int32), xy, sdf, np.zeros(len(xy)), len(xy), len(xy), len(xy),
                         int(np.sum(sdf <= 0)), float(sdf[k]) if k >= 0 else math.inf, k)


def test_repair_bookkeeping():
    pts = np.array([[0.0, 0.0], [0.0, 0.0], [1.0, 1.0]])
    r = plan.Repair(pts)
    a = r.next_points(clearance([[0.0, 0.0], [2.0, 2.0], [3.0, 3.0]], [0.1, -0.2, 0.5]), 3)
    assert np.array_equal(bits(a), bits(np.r_[pts, [[2.0, 2.0], [3.0, 3.0]]]))
    b = r.next_points(clearance([[2.0, 2.0], [4.0, 4.0]], [0.3, 0.6]), 3)
    assert np.array_equal(bits(b), bits(np.r_[a, [[4.0, 4.0]]]))
    assert r.next_points(clearance([[4.0, 4.0]], [0.65]), 3) is None
    s = r.summary()
    assert s["rounds"] == 2 and s["added_per_round"] == [2, 1] and s["stopped"] == "closed"
    assert np.array_equal(bits(s["added"]), bits([[2.0, 2.0], [3.0, 3.0], [4.0, 4.0]]))
    assert s["min_sdf_per_round"] == [-0.2, 0.3, 0.65]
    # the limit: new cells remain after `limit` re-runs
    r = plan.Repair(pts)
    assert r.next_points(clearance([[9.0, 9.0]], [0.0]), 1) is not None
    assert r.next_points(clearance([[8.0, 8.0]], [0.1]), 1) is None
    s = r.summary()
    assert s["rounds"] == 1 and s["stopped"] == "limit" and s["min_sdf_per_round"] == [0.0, 0.1]
    # nothing listed: closed at once, no re-run
    r = plan.Repair(pts)
    assert r.next_points(clearance(np.empty((0, 2)), []), 3) is None
    s = r.summary()
    assert s["rounds"] == 0 and s["added"].shape == (0, 2) and s["stopped"] == "closed" and s["min_sdf_per_round"] == [math.inf]
