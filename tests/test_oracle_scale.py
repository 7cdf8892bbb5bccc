"""Deformable robots on the CPU: the oracle's scaled path (useScale == true, getScale = the project's schedule) against the
reference's own code (tests/golden/ref_pin_scale.npz, written by tests/golden/make_scale_golden.py from
oracle/_ref/libref_path_scaled_*.so), per point and bit for bit, plus the properties the scaled path must have.  The scaled
oracle is oracle/svsdf_oracle_scale.hpp through oracle/scale_py.py."""
import os
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
sys.path.insert(0, GOLD)
import make_scale_golden as mks  # noqa: E402
from oracle import scale_py  # noqa: E402

PAIRS = [("glibc", "glibc"), ("portable", "default")]  # (reference variant, oracle variant)


def bits_differ(a, b):
    a = np.ascontiguousarray(a, dtype=np.float64).ravel()
    b = np.ascontiguousarray(b, dtype=np.float64).ravel()
    assert a.shape == b.shape
    return int((a.view(np.int64) != b.view(np.int64)).sum())


@pytest.fixture(scope="module")
def gscale():
    return np.load(os.path.join(GOLD, "ref_pin_scale.npz"))


def _oracle(O, shape, pp, ov, sched, g):
    """sched None: the rigid oracle (oracle_py.Oracle); otherwise the scaled one."""
    wp, sh, rho = g["params"]
    th = min(8, O.num_procs())
    if sched is None:
        orc = O.Oracle(shape, poly_params=pp, weight_p=wp, safety_hor=sh, rho=rho, threads=th, variant=ov)
    else:
        orc = scale_py.ScaledOracle(shape, sched=sched, poly_params=pp, weight_p=wp, safety_hor=sh, threads=th, variant=ov)
    orc.set_traj(g["T"], g["coeffs"])
    return orc


@pytest.mark.parametrize("sk", list(mks.SCHEDULES))
@pytest.mark.parametrize("rv,ov", PAIRS)
def test_every_shape_matches_scaled_reference_code_bitwise(oracle_mod, gscale, sk, rv, ov):
    g = gscale
    T, co, pts = mks.scene()[:3]
    assert np.array_equal(g["T"], T) and np.array_equal(g["coeffs"], co) and np.array_equal(g["points"], pts)
    pts0 = np.c_[pts, np.zeros(len(pts))]
    n_in = 0
    for ip, pp in enumerate(mks.PRE):
        for s in mks.SHAPES:
            orc = _oracle(oracle_mod, s, pp, ov, mks.SCHEDULES[sk], g)
            sdf, ts, grad, _ = orc.query(pts0)
            key = f"{rv}_{sk}_{ip}_{s}"
            assert bits_differ(sdf, g[key + "_sdf"]) == 0, key
            assert bits_differ(ts, g[key + "_tstar"]) == 0, key
            assert bits_differ(grad, g[key + "_grad"]) == 0, key
            n_in += int((sdf <= 0).sum())
    assert n_in >= 100  # interior (GSIP) points are really exercised
    # the penalty loop: sums equal up to the association order of the additions
    orc = _oracle(oracle_mod, "star", (0.0, 0.0, 0.0), ov, mks.SCHEDULES[sk], g)
    orc.set_points(pts)
    cost, gT, gC, _, _ = orc.cost_grad(T, co)
    rc, rT, rC = float(g[f"{rv}_{sk}_cost"]), g[f"{rv}_{sk}_gradT"], g[f"{rv}_{sk}_gradC"]
    assert abs(cost - rc) <= 1e-13 * abs(rc)
    assert np.linalg.norm(gC - rC) <= 1e-13 * np.linalg.norm(rC)
    assert np.abs(gT - rT).max() <= 1e-12 * np.linalg.norm(rC)


def test_fixture_regenerates_to_the_same_bytes():
    if not scale_py.ref_available():
        pytest.skip("the reference's scaled build exists only where the reference tree does")
    with tempfile.TemporaryDirectory() as d:
        p = mks.generate(os.path.join(d, "again.npz"))
        with open(p, "rb") as a, open(mks.OUT, "rb") as b:
            assert a.read() == b.read()


@pytest.mark.parametrize("ov", ["default", "glibc"])
def test_identity_schedule_is_the_rigid_oracle_bitwise(oracle_mod, gscale, ov):
    g = gscale
    T, co, pts = g["T"], g["coeffs"], g["points"]
    pts0 = np.c_[pts, np.zeros(len(pts))]
    for s in ("star", "sdPie", "fallbackPolygon", "Circle"):
        a = _oracle(oracle_mod, s, (0.3, -0.2, 25.0), ov, mks.SCHEDULES["identity"], g).query(pts0)
        b = _oracle(oracle_mod, s, (0.3, -0.2, 25.0), ov, None, g).query(pts0)
        for x, y in zip(a, b):
            assert bits_differ(x, y) == 0, s
    a = _oracle(oracle_mod, "star", (0.0, 0.0, 0.0), ov, mks.SCHEDULES["identity"], g)
    b = _oracle(oracle_mod, "star", (0.0, 0.0, 0.0), ov, None, g)
    a.set_points(pts)
    b.set_points(pts)
    a.set_threads(1)  # the penalty loop adds in a critical section: one thread fixes the order
    b.set_threads(1)
    ra, rb = a.cost_grad(T, co), b.cost_grad(T, co)
    assert ra[4] == rb[4]
    for x, y in zip(ra[:3], rb[:3]):
        assert bits_differ(x, y) == 0


def _scaled_sdf_at(O, orc, shape, sched, p, t):
    """getSDFAtTimeStamp<true> restated in Python (IEEE double, no contraction): rel = (R^T S^-1)(p - x)."""
    x = orc.traj_pos(t)
    s, c = O.sincos(np.array([x[2]]))
    s, c = float(s[0]), float(c[0])
    _, inv = scale_py.scale_at(sched, t)
    d0, d1 = p[0] - x[0], p[1] - x[1]
    rel = np.array([[(c * inv[0]) * d0 + (s * inv[1]) * d1, (-s * inv[0]) * d0 + (c * inv[1]) * d1, 0.0]])
    return float(O.shape_sdf(shape, rel)[0])


def _scaled_seed(O, orc, shape, sched, p, D):
    """choiceTInit's four layers with the SCALED shape: what the reference would do if the seed scan read useScale."""
    min_dis, seed, dt, t, term = 1e9, 0.0, 0.15, 0.0, D
    for layer in range(1, 5):
        if layer > 1:
            t, term = max(0.0, seed - 10 * dt), min(D, seed + 10 * dt)
        while t <= term:
            f = _scaled_sdf_at(O, orc, shape, sched, p, t)
            if f < min_dis:
                seed, min_dis = t, f
            t += dt
        dt *= 0.1
    return seed


def test_seed_scan_stays_rigid(oracle_mod, gscale):
    """A scaled seed scan would send the descent to another t* on this scene; the reference's (rigid seed) t* is what the
    oracle and the fixture hold."""
    O, g = oracle_mod, gscale
    sched = mks.SCHEDULES["example"]
    orc = _oracle(O, "star", (0.0, 0.0, 0.0), "default", sched, g)
    D = orc.duration()
    pts = g["points"]
    ts_ref = g["portable_example_0_star_tstar"]
    moved = 0
    for k in range(0, len(pts), 2):
        p = np.array([pts[k, 0], pts[k, 1], 0.0])
        seed = _scaled_seed(O, orc, "star", sched, p, D)
        fx, x = orc.gradient_descent(p, max(0.0, seed - 3.4), min(seed + 3.4, D), seed)
        moved += int(x != ts_ref[k])
    assert moved >= 3, moved


def _smoothed_l1(x, mu=0.01):
    if x < 0.0:
        return 0.0
    if x > mu:
        return x - 0.5 * mu
    return (mu - 0.5 * x) * (x / mu) ** 3


def test_gradC_xy_columns_match_finite_differences(oracle_mod, gscale):
    """Outside points, one at a time: the x / y coefficient columns of gradC against central differences of the point's
    penalty w L(safety - sdf) at its t* (t* minimises the sdf over t, so its own motion does not enter; the full cost is
    not used because the reference's descent moves t* in steps).  Moving the trajectory by +delta in x is moving the point
    by -delta, and the column entry of the constant coefficient of the point's piece is dC/dx itself.  The yaw column and
    gradT are not checked: the reference's yaw term omits St^-1 (exact only at St = I) and its gradT follows from it."""
    O, g = oracle_mod, gscale
    sched = mks.SCHEDULES["example"]
    T, co, pts = g["T"], g["coeffs"], g["points"]
    wp, sh, _ = g["params"]
    N = len(T)
    orc = _oracle(O, "star", (0.0, 0.0, 0.0), "default", sched, g)
    sdf, ts, _, _ = orc.query(np.c_[pts, np.zeros(len(pts))])
    sel = np.flatnonzero((sdf > 0.0) & (sdf < sh - 0.02))
    assert sel.size >= 5
    checked = 0
    for k in sel:
        one = _oracle(O, "star", (0.0, 0.0, 0.0), "default", sched, g)
        one.set_points(pts[k:k + 1])
        _, _, gC, pp, _ = one.cost_grad(T, co, per_point=True)
        piece = int(pp[0, 5])
        for d in (0, 1):
            h = 1e-5
            e = np.zeros(3)
            e[d] = h
            cp = wp * _smoothed_l1(sh - _scaled_sdf_at(O, orc, "star", sched, np.r_[pts[k], 0.0] - e, ts[k]))
            cm = wp * _smoothed_l1(sh - _scaled_sdf_at(O, orc, "star", sched, np.r_[pts[k], 0.0] + e, ts[k]))
            fd = (cp - cm) / (2 * h)
            an = gC[d * 6 * N + 6 * piece]
            assert abs(fd - an) <= 1e-3 * max(1.0, abs(an)), (k, d, fd, an)
            checked += 1
    assert checked >= 10
