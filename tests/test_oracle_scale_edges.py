"""Deformable robots at the limits of their inputs, on the CPU: the oracle's scaled path (oracle/svsdf_oracle_scale.hpp through
oracle/scale_py.py) against the reference's own code built with `useScale` on (tests/golden/ref_pin_scale_edges.npz, written by
tests/golden/make_scale_edges_golden.py), per point and bit for bit, on the rigid edge trajectories under edge schedules.

Every (trajectory, schedule) pair is classified by an instrumented restatement of the scaled outer solve (the rigid seed scan,
the scaled descent), which must first reproduce the oracle's outer solve bit for bit.  Each pair asserts the branches it exists
for, so that a later edit to a scene or a schedule cannot silently drop coverage: sin arguments near 1e6 rad, St^-1 near 1e6,
descents with deep halvings and at the 1000-iteration cap, a parked robot flat only under a constant schedule, both velocity
fallback scans and the 9-round cap of the interior branch, t* = 0 and t* = D.  Also: the pinned sin/cos on [1e5, 1e6) against a
60-digit reference, the zero-phase schedule against the rigid oracle, and svsdf_scale_matrix at the accepted limits."""
import os
import sys
import tempfile
from collections import Counter

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
sys.path.insert(0, GOLD)
import make_outer_edges_golden as mko  # noqa: E402
import make_scale_edges_golden as mke  # noqa: E402
from oracle import scale_py  # noqa: E402

CLASSIFY_STRIDE = {"long64": 10}


def bits_differ(a, b):
    """Number of elements whose bit patterns differ."""
    a = np.ascontiguousarray(a, dtype=np.float64).ravel()
    b = np.ascontiguousarray(b, dtype=np.float64).ravel()
    assert a.shape == b.shape
    return int((a.view(np.int64) != b.view(np.int64)).sum())


def inputs(g, name):
    return str(g[f"{name}_shape"]), g[f"{name}_T"], g[f"{name}_coeffs"], g[f"{name}_points"]


def scaled_oracle(O, g, name, sk, variant="default"):
    shape, T, co, _ = inputs(g, name)
    orc = scale_py.ScaledOracle(shape, sched=mke.SCHEDULES[sk], threads=min(8, O.num_procs()), variant=variant)
    orc.set_traj(T, co)
    return orc


@pytest.fixture(scope="module")
def gedge():
    return np.load(os.path.join(GOLD, "ref_pin_scale_edges.npz"))


# ---------------------------------------------------------------------------------------------------------------------
# the fixture
# ---------------------------------------------------------------------------------------------------------------------
def test_fixture_holds_the_scenes_and_schedules(gedge):
    assert list(gedge["schedules"]) == list(mke.SCHEDULES)
    assert np.array_equal(gedge["sched_values"], np.array(list(mke.SCHEDULES.values())))
    for name in mke.MATRIX:
        shape, T, co, pts = mke.scene(name)
        got = inputs(gedge, name)
        assert got[0] == shape and np.array_equal(got[1], T) and np.array_equal(got[2], co) and np.array_equal(got[3], pts), name


@pytest.mark.parametrize("rv,ov", [("portable", "default"), ("glibc", "glibc")])
def test_every_pair_is_bitwise_the_scaled_reference_code(oracle_mod, gedge, rv, ov):
    """query (and, for the portable variant, the outer solve alone) per point, bit for bit, on every (trajectory, schedule)."""
    n_in = 0
    for name, sk in mke.pairs():
        pts = inputs(gedge, name)[3]
        orc = scaled_oracle(oracle_mod, gedge, name, sk, ov)
        sdf, ts, grad, rounds = orc.query(pts)
        key = f"{name}_{sk}_{rv}"
        assert bits_differ(sdf, gedge[key + "_sdf"]) == 0, key
        assert bits_differ(ts, gedge[key + "_tstar"]) == 0, key
        assert bits_differ(grad, gedge[key + "_grad"]) == 0, key
        assert np.all(np.isfinite(sdf)) and np.all(np.isfinite(grad)), key
        if rv == "portable":
            so, to, go = orc.query_outer(pts)
            assert bits_differ(so, gedge[key + "_osdf"]) + bits_differ(to, gedge[key + "_otstar"]) \
                + bits_differ(go, gedge[key + "_ograd"]) == 0, key
            assert np.array_equal(rounds > 0, ~(so > 0)), key
        n_in += int((rounds > 0).sum())
    assert n_in >= 500


def test_fixture_regenerates_to_the_same_bytes():
    if not scale_py.ref_available():
        pytest.skip("the reference's scaled build exists only where the reference tree does")
    with tempfile.TemporaryDirectory() as d:
        p = mke.generate(os.path.join(d, "again.npz"))
        with open(p, "rb") as a, open(mke.OUT, "rb") as b:
            assert a.read() == b.read()


# ---------------------------------------------------------------------------------------------------------------------
# branch classifier: test_gpu_outer_edges.classify_point with the rigid seed scan and the scaled descent
# ---------------------------------------------------------------------------------------------------------------------
def classify_point(orc, sched, p, D, lat):
    """Run choiceTInit (rigid) + gradientDescent (scaled) for one point through orc.sdf_at and record what they did."""
    desc = []

    def f(t):  # the descent's scaled evaluation, at absolute time t
        desc.append(t)
        return orc.sdf_at(p, t, scaled=True)

    min_dis, seed = 1e9, 0.0
    for t in lat:
        d = orc.sdf_at(p, t, scaled=False)
        if d < min_dis:
            min_dis, seed = d, t
    dt = 0.15
    for _layer in range(2, 5):
        dt *= 0.1
        t, term = max(0.0, seed - 10 * dt), min(D, seed + 10 * dt)
        while t <= term:
            d = orc.sdf_at(p, t, scaled=False)
            if d < min_dis:
                seed, min_dis = t, d
            t += dt
    tmin, tmax = max(0.0, seed - 3.4), min(seed + 3.4, D)
    x, prev, it, stop, fx = seed, 10000000.0, 0, False, None
    signs, js = [], []
    while it < 1000 and not stop and abs(x - prev) > 1e-16:
        if it == 0:
            fx = f(x)
        g = (f(min(D, x + 0.000001)) - f(max(0.0, x - 0.000001))) * 500000
        sgn = int(g > 0) - int(g < 0)
        signs.append(sgn)
        tau, prev, acc = 0.01, x, None
        for div in range(1, 30):
            it += 1
            xc = max(min(x + (-tau * sgn), tmax), tmin)
            fc = f(xc)
            if fc - fx < 0:
                x, fx, acc = xc, fc, div - 1
                break
            tau = 0.5 * tau
            if div == 29:
                stop = True
        js.append(acc)
    end = ("zero" if signs[-1] == 0 else "fail29") if stop else ("cap" if it >= 1000 else "tol")
    w, phi = np.array(sched[4:6]), np.array(sched[6:8])
    arg = max(float(np.abs(w * t + phi).max()) for t in desc)
    _, inv = scale_py.scale_at(sched, x)
    return dict(sdf=fx, tstar=x, js=js, end=end, iters=it, arg=arg, inv=float(max(inv[0], inv[1])))


class Pair:
    """One (trajectory, schedule): the oracle's outputs, the interior-branch flags and the classification of its points."""

    def __init__(self, O, g, name, sk):
        self.name, self.sk = name, sk
        self.sched = mke.SCHEDULES[sk]
        shape, self.T, self.co, self.pts = inputs(g, name)
        orc = scaled_oracle(O, g, name, sk)
        self.D = orc.duration()
        self.ref = orc.query(self.pts)
        self.oref = orc.query_outer(self.pts)
        so, to = self.oref[0], self.oref[1]
        inside = ~(so > 0)
        slow = np.zeros(len(self.pts), dtype=bool)
        for k in np.flatnonzero(inside):  # the interior branch's velocity test at the outer t*
            v = orc.traj_vel(to[k])
            slow[k] = np.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]) < 0.01
        self.inside = inside
        self.forward = slow & (to < 0.1)
        self.backward = slow & ~(to < 0.1) & (to > self.D - 0.1)
        lat = mko.lattice(self.D)
        self.cls = {}
        for k in range(0, len(self.pts), CLASSIFY_STRIDE.get(name, 1)):
            c = classify_point(orc, self.sched, self.pts[k], self.D, lat)
            # the restatement is the oracle's outer solve, bit for bit, before anything is read from it
            assert bits_differ(c["sdf"], so[k]) + bits_differ(c["tstar"], to[k]) == 0, (name, sk, k)
            self.cls[k] = c

    def count(self, pred):
        return sum(1 for c in self.cls.values() if pred(c))

    def coverage(self):
        js = [j for c in self.cls.values() for j in c["js"] if j is not None]
        return dict(P=len(self.pts), classified=len(self.cls), inside=int(self.inside.sum()),
                    forward=int(self.forward.sum()), backward=int(self.backward.sum()),
                    nine_rounds=int((self.ref[3] == 9).sum()), tstar_0=int((self.oref[1] == 0.0).sum()),
                    tstar_D=int((self.oref[1] == self.D).sum()), zero_end=self.count(lambda c: c["end"] == "zero"),
                    cap_end=self.count(lambda c: c["end"] == "cap"), max_j=max(js, default=-1),
                    max_iters=max(c["iters"] for c in self.cls.values()),
                    max_arg=max(c["arg"] for c in self.cls.values()), max_inv=max(c["inv"] for c in self.cls.values()))


@pytest.fixture(scope="module")
def classified(oracle_mod, gedge):
    out = {}
    for name, sk in mke.pairs():
        out[name, sk] = p = Pair(oracle_mod, gedge, name, sk)
        print(name, sk, p.coverage())
    return out


def test_every_pair_reaches_what_it_exists_for(classified):
    cov = {k: p.coverage() for k, p in classified.items()}
    # the sin argument sweeps to the top of the Cody-Waite range
    assert cov["long64", "limit_w"]["max_arg"] >= 9e5, cov["long64", "limit_w"]
    # St^-1 near its accepted limit at t*
    for name in mke.MATRIX:
        if "thin" in mke.MATRIX[name]:
            assert cov[name, "thin"]["max_inv"] >= 1e5, (name, cov[name, "thin"])
    # S changing within one descent step: deep accepted halvings and descents at the 1000-iteration cap
    fast = [cov[name, "fast"] for name in mke.MATRIX if "fast" in mke.MATRIX[name]]
    hist = Counter(j for name in mke.MATRIX if "fast" in mke.MATRIX[name]
                   for c in classified[name, "fast"].cls.values() for j in c["js"] if j is not None)
    print("fast: accepted j", dict(sorted(hist.items())))
    assert max(c["max_j"] for c in fast) >= 22, fast
    # the 1000-iteration cap through the scaled descent: no fast pair reaches it (their minima are many and shallow), the spin
    # scene's capped points do under S = I
    assert cov["spin", "zero_phase"]["cap_end"] >= len(mko.SPIN_CAPPED), cov["spin", "zero_phase"]
    # a parked robot: FD slope exactly 0 under a constant schedule, never under a time-varying one
    assert cov["parked", "needle"]["zero_end"] >= 10 and cov["parked", "zero_phase"]["zero_end"] >= 10, cov["parked", "needle"]
    assert cov["parked", "example"]["zero_end"] == 0 and cov["parked", "fast"]["zero_end"] == 0, cov["parked", "example"]
    # the interior branch under a schedule: both velocity fallback scans, the 9-round cap, interior points everywhere
    for sk in ("limit_w", "zero_phase"):  # under "example" and "thin" the scaled outer t* leaves the rest poses
        assert cov["endpoints", sk]["forward"] >= 1 and cov["endpoints", sk]["backward"] >= 1, (sk, cov["endpoints", sk])
    assert max(cov["midstop", sk]["nine_rounds"] for sk in mke.MATRIX["midstop"]) >= 1
    for name in ("endpoints", "midstop", "circle_static", "circle_spin"):
        for sk in mke.MATRIX[name]:
            assert cov[name, sk]["inside"] >= 1, (name, sk, cov[name, sk])
    # both ends of the trajectory as t*
    assert sum(c["tstar_0"] for c in cov.values()) >= 1 and sum(c["tstar_D"] for c in cov.values()) >= 1
    for sk in ("limit_w", "fast", "thin", "pi_phase"):  # under "example" t* leaves the start of tiny_n2
        assert cov["tiny_n2", sk]["tstar_0"] >= 1 and cov["tiny_n2", sk]["tstar_D"] >= 1, (sk, cov["tiny_n2", sk])


def test_zero_phase_is_the_rigid_oracle_and_pi_phase_is_not(oracle_mod, gedge):
    """sin(0) = 0 with a = 1 gives S = I exactly: the rigid oracle's bits.  sin(pi) ~ 1.2e-16 times b = 0.95 moves S off I by
    one ulp: not the rigid oracle's bits somewhere, bit for bit the reference's (above)."""
    for sk, want_equal in (("zero_phase", True), ("pi_phase", False)):
        differ = 0
        for name in mke.MATRIX:
            if sk not in mke.MATRIX[name]:
                continue
            shape, T, co, pts = inputs(gedge, name)
            rig = oracle_mod.Oracle(shape, threads=min(8, oracle_mod.num_procs()))
            rig.set_traj(T, co)
            a = scaled_oracle(oracle_mod, gedge, name, sk).query(pts)
            b = rig.query(pts)
            differ += sum(bits_differ(x, y) for x, y in zip(a[:3], b[:3]))
        assert (differ == 0) == want_equal, (sk, differ)


# ---------------------------------------------------------------------------------------------------------------------
# the pinned sin/cos where the schedule's arguments end: [1e5, 1e6)
# ---------------------------------------------------------------------------------------------------------------------
def hard_arguments(n, lo=1e5, hi=1e6):
    """The n doubles in [lo, hi) closest to a multiple of pi/2 (smallest |x - k pi/2|, the largest cancellation in the
    reduction), found with exact integer arithmetic: pi/2 from Machin's formula to 300 bits (as _two_over_pi_words in
    tests/test_portable_math.py), and for every multiple k pi/2 in range the double nearest to it."""
    bits = 300
    one = 1 << bits

    def arctan_inv(k):  # arctan(1/k) * 2^bits, truncated term by term
        s, t, j, sign = 0, one // k, 1, 1
        while t:
            s += sign * (t // j)
            t //= k * k
            j += 2
            sign = -sign
        return s

    half_pi = (16 * arctan_inv(5) - 4 * arctan_inv(239)) // 2  # pi/2 * 2^bits, a few units off in the last place
    out = []
    for k in range((int(lo) << bits) // half_pi, (int(hi) << bits) // half_pi + 1):
        m = k * half_pi
        e = (m >> bits).bit_length() - 53  # ulp of the doubles around k pi/2 is 2^e (>= 2^-36 here)
        unit = 1 << (bits + e)
        q = (m + unit // 2) // unit  # nearest double, in ulps
        x = q * 2.0**e
        if lo <= x < hi:
            out.append((abs(q * unit - m), x))
    out.sort()
    return np.array([x for _, x in out[:n]])


def test_portable_sincos_below_1e6_is_within_2ulp_of_60_digits(oracle_mod):
    """The Cody-Waite range of the pinned sin/cos, where svsdf_set_scale keeps the schedule's arguments: 20 000 random
    arguments and the 2 000 doubles closest to a multiple of pi/2 (where the reduced argument, and so the relative error of
    cos or sin, is smallest and the reduction's cancellation largest), against mpmath at 60 digits."""
    import mpmath

    mpmath.mp.dps = 60
    rng = np.random.default_rng(71)
    hard = hard_arguments(2000)
    assert len(hard) == 2000 and hard.min() >= 1e5 and hard.max() < 1e6
    x = np.concatenate([rng.uniform(1e5, 1e6, 20_000), hard, -hard[:200], [1e5, np.nextafter(1e6, 0)]])
    s, c = oracle_mod.sincos(x)
    worst = {}
    for name, got, fn in (("sin", s, mpmath.sin), ("cos", c, mpmath.cos)):
        err = np.empty(len(x))
        for i, xi in enumerate(x):
            exact = fn(mpmath.mpf(float(xi)))
            err[i] = float(abs(mpmath.mpf(float(got[i])) - exact) / mpmath.mpf(float(np.spacing(abs(float(exact))))))
        worst[name] = (float(err.max()), float(x[err.argmax()]), float(err[20_000:22_000].max()))
    print("sincos on [1e5, 1e6): worst ulp (all, argument, hard only)", worst)
    assert worst["sin"][0] <= 2.0 and worst["cos"][0] <= 2.0, worst


# ---------------------------------------------------------------------------------------------------------------------
# svsdf_scale_matrix at the accepted limits (no GPU needed)
# ---------------------------------------------------------------------------------------------------------------------
REFUSED = [
    dict(a=(1e-160, 1e-160)),                       # a - |b| > 0, but fl(sy sx) is subnormal: 1/det = inf
    dict(a=(1e160, 1e160)),                         # fl(sy sx) = inf: St^-1 = 0, S^-1's (3,3) entry inf * 0 = NaN
    dict(a=(1.0, 1.0), b=(0.9999995, 0.0)),         # a - |b| = 5e-7: just below the lower bound
    dict(a=(1.0, 5e-7)),
    dict(a=(1e6, 1.0), b=(1e-9, 0.0)),              # a + |b| just above the upper bound
    dict(a=(1.0, 2e6)),
    dict(a=(5e5, 1.0), b=(-5e5, 0.0)),              # a - |b| = 0
]
ACCEPTED = [
    dict(a=(1.0, 1.0), b=(0.999999, 0.0)),          # a - |b| = 1.00000000003e-6
    dict(a=(1e-6, 1e-6)),
    dict(a=(1e6, 1e6)),
    dict(a=(1.0, 5e5), b=(0.0, -5e5 + 1e-6)),       # s_y from 1e-6 to 1e6 within one period
]


@pytest.mark.parametrize("bad", REFUSED, ids=lambda d: ",".join(f"{k}={v}" for k, v in d.items()))
def test_scale_matrix_refuses_schedules_with_no_finite_inverse(bad):
    from implicit_svsdf_planner_b200 import api

    with pytest.raises(api.SvsdfError):
        api.scale_matrix(0.0, **bad)


def test_scale_matrix_at_the_bounds_is_finite_and_the_oracles():
    """At both bounds and at the fixture's schedules, over t in [0, 300]: S and St^-1 finite and non-zero on the diagonal, and
    bit for bit the oracle's scale_at (the reference's arithmetic).  Just inside the bounds the unvalidated arithmetic is
    what the refused cases above show it is not: finite."""
    from implicit_svsdf_planner_b200 import api

    ts = np.r_[np.linspace(0.0, 300.0, 301), 299.84, 1.2345]
    scheds = [dict(a=d["a"], b=d.get("b", (0.0, 0.0)), w=(0.0, 0.3)) for d in ACCEPTED]
    scheds += [dict(a=v[0:2], b=v[2:4], w=v[4:6], phi=v[6:8]) for v in mke.SCHEDULES.values()]
    for z in scheds:
        flat = (*z["a"], *z.get("b", (0.0, 0.0)), *z.get("w", (0.0, 0.0)), *z.get("phi", (0.0, 0.0)))
        for t in ts:
            S, Si = api.scale_matrix(t, **z)
            s2, inv3 = scale_py.scale_at(flat, t)
            assert np.all(np.isfinite(S)) and np.all(np.isfinite(Si)), (z, t)
            assert np.all(np.diag(Si) != 0.0), (z, t)
            assert bits_differ(np.diag(S)[:2], s2) + bits_differ(np.diag(Si), inv3) == 0, (z, t)
    # what the refused cases compute in the reference's arithmetic: not finite
    for d in REFUSED[:2]:
        _, inv3 = scale_py.scale_at((*d["a"], 0.0, 0.0, 0.0, 0.0, 0.0, 0.0), 0.0)
        assert not np.all(np.isfinite(inv3)) or np.any(inv3 == 0.0), (d, inv3)
