"""CPU tests of tests/reduction_ref.py, the restatement of the cost path's last stage (point_contribution and the reduction
of its terms into cost, gradC and gradT).

The oracle's penalty loop (oracle/svsdf_oracle.hpp, addSafetyPenaltyTrueSDF) run with one thread adds the points in order,
and its per-point records are pinned on the reference's own code (tests/test_oracle_ref_pin.py).  So:
  * point_terms fed with the oracle's per-point record reproduces its piece and penalty bit for bit, and fed with the oracle's
    query outputs (world-frame GSIP direction at interior points, what svsdf_query returns) the same terms;
  * those terms summed in the oracle's order reproduce the oracle's cost, gradC and gradT bit for bit;
  * exact_record lies within gamma_P of the oracle's sequential sums and within gamma_bound of ordered_record for several
    schedules (a self-consistency check of the helper the GPU tests rely on).
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import scenes

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_outer_edges_golden as mko  # noqa: E402
import make_scale_golden as mks  # noqa: E402
import reduction_ref as R  # noqa: E402

SCHED = {k: dict(a=v[0:2], b=v[2:4], w=v[4:6], phi=v[6:8]) for k, v in mks.SCHEDULES.items()}


def _scene(name):
    """(shape, T, coeffs, points, weight_p, safety_hor)"""
    if name == "scene2k":
        sc = scenes.make_scene("star", 8, 2000)
    elif name == "small_inside":
        sc = scenes.make_scene("star", 8, 400, clearance=2.35)
    elif name == "n1":
        shape, T, co, pts = mko.scene("tiny_k1")
        return shape, T, co, pts, 60.0, 0.7
    elif name == "n64":
        shape, T, co, pts = mko.scene("long64")
        return shape, T, co, pts[::4], 60.0, 0.7
    else:
        raise KeyError(name)
    return "star", sc.T, sc.coeffs_colmajor(), sc.points, sc.weight_p, sc.safety_hor


def _oracle_run(oracle_mod, name, sched=None):
    shape, T, co, pts, wp, sh = _scene(name)
    if sched is None:
        orc = oracle_mod.Oracle(shape, weight_p=wp, safety_hor=sh, threads=1)
    else:
        from oracle import scale_py

        orc = scale_py.ScaledOracle(shape, sched=mks.SCHEDULES[sched], weight_p=wp, safety_hor=sh, threads=1)
    orc.set_points(pts)
    c, gT, gC, pp, n_in = orc.cost_grad(T, co, per_point=True)
    orc.set_traj(T, co)
    q = orc.query(np.c_[pts[:, :2], np.zeros(len(pts))])
    N = len(T)
    return dict(T=T, co=co, pts=pts, wp=wp, sh=sh, N=N, rec=np.r_[c, gC, gT], pp=pp, n_in=n_in, query=q,
                scale=None if sched is None else SCHED[sched])


CASES = [("scene2k", None), ("small_inside", None), ("n1", None), ("n64", None), ("small_inside", "example"),
         ("small_inside", "aniso")]


@pytest.fixture(scope="module", params=CASES, ids=[f"{a}-{b or 'rigid'}" for a, b in CASES])
def run(request, oracle_mod):
    return _oracle_run(oracle_mod, *request.param)


def test_terms_reproduce_the_oracles_per_point_records(run):
    pp = run["pp"]
    tr = R.point_terms(run["pts"], run["T"], run["co"], pp[:, 0], pp[:, 1], pp[:, 2:4], run["wp"], run["sh"],
                       scale=run["scale"], rotate_interior=False)
    assert np.array_equal(tr.piece, pp[:, 5].astype(np.int64))
    assert R.bits_equal(tr.pena + 0.0, pp[:, 6] + 0.0)  # the oracle accumulates pena from +0.0
    assert tr.active.sum() > 0


def test_terms_from_query_outputs_rotate_the_interior_direction(run):
    """svsdf_query's outputs (the oracle's query: world-frame GSIP direction inside) give the same terms once point_terms rotates
    them where sdf < 0; without the rotation the interior terms differ."""
    pp = run["pp"]
    sdf, ts, g, _ = run["query"]
    assert R.bits_equal(sdf, pp[:, 0]) and R.bits_equal(ts, pp[:, 1])
    a = R.point_terms(run["pts"], run["T"], run["co"], sdf, ts, g, run["wp"], run["sh"], scale=run["scale"])
    b = R.point_terms(run["pts"], run["T"], run["co"], pp[:, 0], pp[:, 1], pp[:, 2:4], run["wp"], run["sh"], scale=run["scale"],
                      rotate_interior=False)
    assert R.bits_equal(a.gc, b.gc) and R.bits_equal(a.gdT, b.gdT) and R.bits_equal(a.pena, b.pena)
    if (sdf < 0).any():
        c = R.point_terms(run["pts"], run["T"], run["co"], sdf, ts, g, run["wp"], run["sh"], scale=run["scale"],
                          rotate_interior=False)
        assert not R.bits_equal(c.gc, a.gc)


def test_oracle_order_reproduces_the_oracle_bit_for_bit(run):
    pp = run["pp"]
    tr = R.point_terms(run["pts"], run["T"], run["co"], pp[:, 0], pp[:, 1], pp[:, 2:4], run["wp"], run["sh"],
                       scale=run["scale"], rotate_interior=False)
    rec = R.oracle_order_record(tr)
    assert R.bits_equal(rec, run["rec"]), np.flatnonzero(rec != run["rec"])[:10]


def test_exact_record_bounds_both_orders(run):
    """exact_record is within gamma_P of the oracle's sequential sums (every chain at most P long) and within gamma_bound of
    ordered_record for sparse and batched schedules on 1, 3, 37 and 396 CTAs."""
    pp = run["pp"]
    N = run["N"]
    tr = R.point_terms(run["pts"], run["T"], run["co"], pp[:, 0], pp[:, 1], pp[:, 2:4], run["wp"], run["sh"],
                       scale=run["scale"], rotate_interior=False)
    ex, ab = R.exact_record(tr)
    P = len(run["pts"])
    assert (np.abs(run["rec"] - ex) <= R.gamma(P) * ab).all()
    # the kernels' interior flag: the outer solve's sdf <= 0, i.e. a GSIP round count > 0 (the oracle counts the final sdf <= 0,
    # which differs where the interior branch ends with r* < 0)
    inside = run["query"][3] > 0
    assert (inside | (pp[:, 0] > 0)).all() and inside.sum() >= run["n_in"]
    for grid in (1, 3, 37, 396):
        for batched in (None, False, True):
            out, info = R.ordered_record(tr, inside, grid, batched)
            assert out[-1] == inside.sum()
            err = np.abs(out[:-1] - ex)
            assert (err <= R.gamma_bound(info, ab, N)).all(), (grid, batched, info)
            # gradT: the last entry is the empty suffix
            assert R.bits_equal(out[1 + 19 * N - 1], 0.0)


def test_smoothed_l1_is_the_oracles(oracle_mod):
    L = oracle_mod.lib()
    L.orc_smoothed_l1.argtypes = [C.c_int64, C.POINTER(C.c_double), C.c_double, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                  C.POINTER(C.c_uint8)]
    rng = np.random.default_rng(11)
    mu = 0.01
    x = np.r_[-1.0, -1e-300, -0.0, 0.0, 5e-324, 1e-300, rng.uniform(0.0, mu, 20000), mu * 0.5, np.nextafter(mu, 0.0), mu,
              np.nextafter(mu, 1.0), rng.uniform(mu, 10.0, 5000), 0.7, 1e300]
    f, df, ret = np.full(x.size, -1.0), np.zeros(x.size), np.zeros(x.size, dtype=np.uint8)
    dp = C.POINTER(C.c_double)
    L.orc_smoothed_l1(x.size, x.ctypes.data_as(dp), mu, f.ctypes.data_as(dp), df.ctypes.data_as(dp), ret.ctypes.data_as(C.POINTER(C.c_uint8)))
    r2, f2, df2 = R.smoothed_l1(x, mu)
    assert np.array_equal(r2, ret.astype(bool))
    assert R.bits_equal(f2[r2], f[r2]) and R.bits_equal(df2[r2], df[r2])
    assert not r2[0] and r2[2] and r2[3]  # x < 0 only is rejected; -0.0 is not < 0


def test_locate_piece_is_the_subtraction_chain():
    T = np.array([0.3, 0.1, 0.2])
    D = 0.0
    for d in T:
        D += d
    t = np.array([0.0, 0.3, np.nextafter(0.3, 1.0), 0.4, D, D + 1.0, -1.0, np.nan])
    piece, tl = R.locate_piece(T, t)
    for k, tk in enumerate(t):
        j, x = 0, tk
        while j < len(T) and x > T[j]:
            x -= T[j]
            j += 1
        if j == len(T):
            j -= 1
            x += T[j]
        assert piece[k] == j and R.bits_equal(tl[k], x), (tk, piece[k], j)
    assert piece[5] == 2 and piece[4] == 2  # t >= D: clamped to the last piece


def test_ordered_record_edge_schedules():
    """P = 0 gives +0.0 everywhere; a single active point passes through every stage unchanged (each addition starts from
    +0.0); the schedules cover every point exactly once."""
    for P, grid, batched in ((0, 1, False), (1, 1, False), (33, 5, True), (1000, 3, True), (1000, 7, False), (2000, 396, True)):
        sch = R.warp_schedule(P, grid, batched)
        got = np.sort(sch[sch >= 0])
        assert np.array_equal(got, np.arange(P)), (P, grid, batched)
    tr = R.Terms(piece=np.zeros(0, dtype=np.int64), s1=np.zeros(0), G=np.zeros((0, 3)), gc=np.zeros((0, 3, 6)), gdT=np.zeros(0),
                 pena=np.zeros(0), active=np.zeros(0, dtype=bool), B=np.zeros((0, 20)), N=3)
    out, info = R.ordered_record(tr, np.zeros(0, dtype=bool), 1)
    assert R.bits_equal(out, np.zeros(1 + 19 * 3 + 1))
    rng = np.random.default_rng(3)
    gc = rng.normal(size=(1, 3, 6))
    tr = R.Terms(piece=np.array([1]), s1=np.array([0.5]), G=gc[:, :, 0], gc=gc, gdT=np.array([-2.5]), pena=np.array([3.0]),
                 active=np.array([True]), B=np.ones((1, 20)), N=3)
    for inside in (False, True):
        out, _ = R.ordered_record(tr, np.array([inside]), 1)
        assert out[0] == 3.0 and out[-1] == float(inside)
        assert R.bits_equal(out[1 + 18 * 3:1 + 19 * 3], [-2.5, 0.0, 0.0])
        assert R.bits_equal(out[R._acc_index(3)[18:36]], gc[0].reshape(18))
