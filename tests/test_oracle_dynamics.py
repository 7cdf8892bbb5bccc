"""CPU: the back end's speed and yaw-rate penalty (svsdf_dynamics_penalty, host::dynamics_penalty in csrc/host/minco.hpp) against a
plain-Python restatement of its definition, bit for bit in the documented summation order; its gradient against central
differences; limits never reached; and the inputs it refuses."""
import ctypes as C
import math

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api


def smoothed_l1(x, mu):
    """back_end_optimizer.hpp:316-340: None below 0, else (f, df)."""
    if x < 0.0:
        return None
    if x > mu:
        return x - 0.5 * mu, 1.0
    xdmu = x / mu
    sqrxdmu = xdmu * xdmu
    mumxd2 = mu - 0.5 * x
    return mumxd2 * sqrxdmu * xdmu, sqrxdmu * ((-0.5) * xdmu + 3.0 * mumxd2 / mu)


def penalty_ref(d, T, b, regions=None):
    """The penalty as the header defines it, operation for operation.  d: dict of the limits; b: 18N column-major.  regions (a dict)
    counts the samples of each violation below 0, in [0, mu] and above mu.  Returns (cost, gradT, gradC)."""
    N = len(T)
    n = 6 * N
    res = d["integralIntervs"]
    mu = d["smoothingEps"]
    vs, os_ = d["vmax"] * d["vmax"], d["omgmax"] * d["omgmax"]
    frac = 1.0 / res
    gC, gT, partial = [0.0] * (18 * N), [0.0] * N, [0.0] * N
    for i in range(N):
        step = float(T[i]) * frac
        c = [[float(b[dd * n + 6 * i + k]) for k in range(6)] for dd in range(3)]
        part = 0.0
        for j in range(res + 1):
            s1 = j * step
            s2 = s1 * s1
            s3 = s2 * s1
            s4 = s2 * s2
            vel = [c[dd][1] + 2.0 * s1 * c[dd][2] + 3.0 * s2 * c[dd][3] + 4.0 * s3 * c[dd][4] + 5.0 * s4 * c[dd][5] for dd in range(3)]
            viola_v = vel[0] * vel[0] + vel[1] * vel[1] - vs
            viola_o = vel[2] * vel[2] - os_
            if regions is not None:
                for name, x in (("v", viola_v), ("omg", viola_o)):
                    key = name + ("<0" if x < 0 else ("<=mu" if x <= mu else ">mu"))
                    regions[key] = regions.get(key, 0) + 1
            gv, pena, active = [0.0, 0.0, 0.0], 0.0, False
            r = smoothed_l1(viola_v, mu)
            if r is not None:
                f, df = r
                gv[0] = d["weight_v"] * df * 2.0 * vel[0]
                gv[1] = d["weight_v"] * df * 2.0 * vel[1]
                pena += d["weight_v"] * f
                active = True
            r = smoothed_l1(viola_o, mu)
            if r is not None:
                f, df = r
                gv[2] = d["weight_omg"] * df * 2.0 * vel[2]
                pena += d["weight_omg"] * f
                active = True
            if not active:
                continue
            node = 0.5 if (j == 0 or j == res) else 1.0
            alpha = j * frac
            dot = 0.0
            for dd in range(3):
                cc = c[dd]
                acc = 2.0 * cc[2] + 6.0 * s1 * cc[3] + 12.0 * s2 * cc[4] + 20.0 * s3 * cc[5]
                dot = gv[0] * acc if dd == 0 else dot + gv[dd] * acc
                o = dd * n + 6 * i
                gC[o + 1] += 1.0 * gv[dd] * node * step
                gC[o + 2] += 2.0 * s1 * gv[dd] * node * step
                gC[o + 3] += 3.0 * s2 * gv[dd] * node * step
                gC[o + 4] += 4.0 * s3 * gv[dd] * node * step
                gC[o + 5] += 5.0 * s4 * gv[dd] * node * step
            gT[i] += dot * alpha * node * step + node * frac * pena
            part += node * step * pena
        partial[i] = part
    cost = 0.0
    for i in range(N):  # the partials in ascending piece order
        cost += partial[i]
    return cost, np.array(gT), np.array(gC)


def lib_penalty(d, T, b):
    return api.dynamics_penalty(T, b, d)


def random_traj(rng, N, tmin=0.001, tmax=20.0, speed=1.0):
    """Durations log-uniform in [tmin, tmax] (both ends included for N >= 2) and coefficients whose velocity scale is about `speed`
    over each piece, yaw rates of either sign."""
    T = np.exp(rng.uniform(math.log(tmin), math.log(tmax), N))
    if N >= 2:
        T[0], T[-1] = tmin, tmax
    b = np.zeros((3, N, 6))
    for i in range(N):
        for k in range(6):
            # |c_k s^(k-1) k| ~ speed at s = T_i
            b[:, i, k] = rng.normal(0.0, 1.0, 3) * speed / (max(k, 1) * T[i] ** max(k - 1, 0))
    return T, b.reshape(-1)


def limits(**kw):
    d = api.dynamics().as_dict()
    d.update(kw)
    return d


def assert_bits(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), np.flatnonzero(a.view(np.uint64) != b.view(np.uint64))[:10]


def speed_quantiles(d, T, b):
    """vmax / omgmax that put the restatement's samples on every side of the smoothing band: the limits are set at a median speed,
    and one sample's violation is moved into [0, mu]."""
    res = d["integralIntervs"]
    N = len(T)
    c = np.asarray(b).reshape(3, N, 6)
    v2, w2 = [], []
    for i in range(N):
        for j in range(res + 1):
            s = j * (T[i] * (1.0 / res))
            vel = [c[dd, i, 1] + 2 * s * c[dd, i, 2] + 3 * s * s * c[dd, i, 3] + 4 * s ** 3 * c[dd, i, 4] + 5 * s ** 4 * c[dd, i, 5]
                   for dd in range(3)]
            v2.append(vel[0] ** 2 + vel[1] ** 2)
            w2.append(vel[2] ** 2)
    v2, w2 = np.sort(v2), np.sort(w2)
    return v2, w2


CASES = [(N, res, seed) for N in (1, 2, 8, 64) for res in (1, 4, 64) for seed in (0, 1)]


@pytest.mark.parametrize("N,res,seed", CASES)
def test_penalty_is_the_restatement_bit_for_bit(N, res, seed):
    rng = np.random.default_rng(1000 * N + 10 * res + seed)
    T, b = random_traj(rng, N)
    d = limits(integralIntervs=res, weight_v=7.5, weight_omg=3.25)
    v2, w2 = speed_quantiles(d, T, b)
    # mu: 1e-2 (the yaml's) or a tenth of the samples' spread around the median, whichever is smaller
    m = len(v2) // 2
    spread = min(v2[m] - v2[m // 2], v2[(m + len(v2)) // 2] - v2[m], w2[m] - w2[m // 2], w2[(m + len(w2)) // 2] - w2[m])
    few = N * (res + 1) < 16
    mu = d["smoothingEps"] = 1e-2 if few or spread <= 0 else (min(1e-2, 0.1 * spread) if seed == 1 else 0.1 * spread)
    # the median sample sits inside [0, mu] (violation mu / 2 before rounding), half the samples below 0, half above
    d["vmax"] = math.sqrt(max(v2[len(v2) // 2] - 0.5 * mu, 1e-300))
    d["omgmax"] = math.sqrt(max(w2[len(w2) // 2] - 0.5 * mu, 1e-300))
    regions = {}
    ref = penalty_ref(d, T, b, regions)
    got = lib_penalty(d, T, b)
    assert_bits(got[0], ref[0])
    assert_bits(got[1], ref[1])
    assert_bits(got[2], ref[2])
    if not few:  # enough samples for every region of both violations
        for key in ("v<0", "v<=mu", "v>mu", "omg<0", "omg<=mu", "omg>mu"):
            assert regions.get(key, 0) > 0, (key, regions)
    assert got[0] > 0.0


def test_negative_yaw_rates_and_extreme_durations_are_covered():
    rng = np.random.default_rng(7)
    T, b = random_traj(rng, 64)
    c = b.reshape(3, 64, 6)
    assert (c[2, :, 1] < 0).any() and (c[2, :, 1] > 0).any()  # yaw rates of both signs at s = 0
    assert T.min() == 0.001 and T.max() == 20.0
    d = limits(vmax=0.5, omgmax=0.5, integralIntervs=4)
    ref = penalty_ref(d, T, b)
    got = lib_penalty(d, T, b)
    for a, r in zip(got, ref):
        assert_bits(a, r)


def test_sum_is_per_piece_partials_in_piece_order():
    """The cost is the sum of per-piece partials, not one running sum over every sample: on this trajectory the two orders differ."""
    rng = np.random.default_rng(3)
    T, b = random_traj(rng, 64)
    d = limits(vmax=0.3, omgmax=0.3, integralIntervs=64, smoothingEps=1e-3)
    got = lib_penalty(d, T, b)[0]
    assert_bits(got, penalty_ref(d, T, b)[0])
    # the sample-order sum of the same terms
    N, res, frac = 64, 64, 1.0 / 64
    ref_sample_order = 0.0
    c = b.reshape(3, N, 6)
    for i in range(N):
        step = T[i] * frac
        for j in range(res + 1):
            s1 = j * step
            s2, s3, s4 = s1 * s1, s1 * s1 * s1, (s1 * s1) * (s1 * s1)
            vel = [c[k, i, 1] + 2.0 * s1 * c[k, i, 2] + 3.0 * s2 * c[k, i, 3] + 4.0 * s3 * c[k, i, 4] + 5.0 * s4 * c[k, i, 5] for k in range(3)]
            pena = 0.0
            r = smoothed_l1(vel[0] * vel[0] + vel[1] * vel[1] - d["vmax"] * d["vmax"], d["smoothingEps"])
            if r is not None:
                pena += d["weight_v"] * r[0]
            r = smoothed_l1(vel[2] * vel[2] - d["omgmax"] * d["omgmax"], d["smoothingEps"])
            if r is not None:
                pena += d["weight_omg"] * r[0]
            node = 0.5 if (j == 0 or j == res) else 1.0
            ref_sample_order += node * step * pena
    assert ref_sample_order != got


def _fd_case(seed, N, res):
    rng = np.random.default_rng(seed)
    T, b = random_traj(rng, N, tmin=0.2, tmax=3.0)
    mu = 1e-4
    d = limits(integralIntervs=res, smoothingEps=mu, weight_v=2.0, weight_omg=5.0)
    v2, w2 = speed_quantiles(d, T, b)
    # limits between two samples' speeds, far from every sample in units of mu
    for key, arr in (("vmax", v2), ("omgmax", w2)):
        gaps = np.diff(arr)
        k = int(np.argmax(gaps[len(gaps) // 4: 3 * len(gaps) // 4])) + len(gaps) // 4
        d[key] = math.sqrt(0.5 * (arr[k] + arr[k + 1]) - 0.5 * mu)
    return d, T, b


def _violations(d, T, b):
    regions, out = {}, []
    N, res = len(T), d["integralIntervs"]
    c = b.reshape(3, N, 6)
    for i in range(N):
        step = T[i] * (1.0 / res)
        for j in range(res + 1):
            s = j * step
            vel = [c[k, i, 1] + 2 * s * c[k, i, 2] + 3 * s * s * c[k, i, 3] + 4 * s ** 3 * c[k, i, 4] + 5 * s ** 4 * c[k, i, 5] for k in range(3)]
            out += [vel[0] ** 2 + vel[1] ** 2 - d["vmax"] ** 2, vel[2] ** 2 - d["omgmax"] ** 2]
    return np.array(out)


@pytest.mark.parametrize("seed,N,res", [(11, 2, 4), (12, 8, 4), (13, 8, 16), (14, 1, 8)])
def test_gradient_matches_central_differences(seed, N, res):
    d, T, b = _fd_case(seed, N, res)
    mu = d["smoothingEps"]
    viol = _violations(d, T, b)
    assert np.all((viol <= -10 * mu) | (viol >= 11 * mu)), np.min(np.abs(viol))
    assert (viol > 0).any()
    cost, gT, gC = lib_penalty(d, T, b)
    assert cost > 0

    def f(TT, bb):
        return lib_penalty(d, TT, bb)[0]

    scale = max(np.abs(gC).max(), np.abs(gT).max())
    for e in range(18 * N):
        h = 1e-6 * max(1.0, abs(b[e]))
        bp, bm = b.copy(), b.copy()
        bp[e] += h
        bm[e] -= h
        fd = (f(T, bp) - f(T, bm)) / (2 * h)
        assert abs(fd - gC[e]) <= 1e-6 * max(abs(gC[e]), 1e-3 * scale), (e, fd, gC[e])
    for i in range(N):
        h = 1e-7 * T[i]
        Tp, Tm = T.copy(), T.copy()
        Tp[i] += h
        Tm[i] -= h
        fd = (f(Tp, b) - f(Tm, b)) / (2 * h)
        assert abs(fd - gT[i]) <= 1e-6 * max(abs(gT[i]), 1e-3 * scale), (i, fd, gT[i])
    # the central differences are only valid where no violation crosses 0 or mu within a step
    assert np.all((_violations(d, T, b * (1 + 1e-6)) <= 0) == (viol <= 0))


def test_limits_never_reached_give_zero():
    rng = np.random.default_rng(5)
    for N in (1, 8, 64):
        T, b = random_traj(rng, N, tmin=0.5, tmax=2.0, speed=0.1)
        d = limits(vmax=1e6, omgmax=1e6, integralIntervs=8)
        cost, gT, gC = lib_penalty(d, T, b)
        assert cost == 0.0
        assert not gT.any() and not gC.any()


def _raw(d, N, T, b, cost, gC, gT):
    dd = api.dynamics(d) if d is not None else None
    return api.lib().svsdf_dynamics_penalty(C.byref(dd) if dd is not None else None, N, api._p(T) if T is not None else None,
                                           api._p(b) if b is not None else None, api._p(cost) if cost is not None else None,
                                           api._p(gC) if gC is not None else None, api._p(gT) if gT is not None else None)


BAD_LIMITS = [dict(vmax=0.0), dict(vmax=-1.0), dict(omgmax=0.0), dict(omgmax=-2.0), dict(weight_v=-1e-9), dict(weight_omg=-1.0),
              dict(smoothingEps=0.0), dict(smoothingEps=-1e-2), dict(integralIntervs=0), dict(integralIntervs=65), dict(integralIntervs=-3),
              dict(vmax=math.inf), dict(omgmax=math.nan), dict(weight_v=math.inf), dict(weight_omg=math.nan), dict(smoothingEps=math.inf)]


@pytest.mark.parametrize("bad", BAD_LIMITS, ids=[",".join(f"{k}={v}" for k, v in b.items()) for b in BAD_LIMITS])
def test_refused_limits_write_nothing(bad):
    rng = np.random.default_rng(9)
    N = 4
    T, b = random_traj(rng, N)
    cost, gC, gT = np.full(1, 7.0), np.full(18 * N, 7.0), np.full(N, 7.0)
    assert _raw(limits(**bad), N, T, b, cost, gC, gT) == -1
    assert (cost == 7.0).all() and (gC == 7.0).all() and (gT == 7.0).all()
    with pytest.raises(api.SvsdfError):
        api.dynamics_penalty(T, b, limits(**bad))


def test_refused_arguments_write_nothing():
    rng = np.random.default_rng(10)
    N = 3
    T, b = random_traj(rng, N)
    d = limits()
    for args in [(None, N, T, b), (d, 0, T, b), (d, -1, T, b), (d, N, None, b), (d, N, T, None)]:
        cost, gC, gT = np.full(1, 7.0), np.full(18 * N, 7.0), np.full(N, 7.0)
        assert _raw(*args, cost, gC, gT) == -1
        assert (cost == 7.0).all() and (gC == 7.0).all() and (gT == 7.0).all()
    for outs in [(None, np.zeros(18 * N), np.zeros(N)), (np.zeros(1), None, np.zeros(N)), (np.zeros(1), np.zeros(18 * N), None)]:
        keep = [o.copy() if o is not None else None for o in outs]
        assert _raw(d, N, T, b, *outs) == -1
        for o, k in zip(outs, keep):
            if o is not None:
                assert_bits(o, k)
    # the edges of the valid range are accepted
    for ok in (dict(integralIntervs=1), dict(integralIntervs=64), dict(weight_v=0.0, weight_omg=0.0), dict(smoothingEps=1e-300)):
        assert _raw(limits(**ok), N, T, b, np.zeros(1), np.zeros(18 * N), np.zeros(N)) == 0


def test_outputs_are_overwritten_not_accumulated():
    rng = np.random.default_rng(12)
    N = 5
    T, b = random_traj(rng, N)
    d = limits(vmax=0.2, omgmax=0.2)
    cost, gC, gT = np.full(1, 3.0), np.full(18 * N, 3.0), np.full(N, 3.0)
    assert _raw(d, N, T, b, cost, gC, gT) == 0
    ref = penalty_ref(d, T, b)
    assert_bits(cost[0], ref[0])
    assert_bits(gT, ref[1])
    assert_bits(gC, ref[2])


def test_yaml_dynamics_and_defaults():
    from implicit_svsdf_planner_b200 import scenes

    d = api.yaml_dynamics(scenes.YAML).as_dict()
    assert d == dict(vmax=10.0, omgmax=10.0, weight_v=10.0, weight_omg=10.0, smoothingEps=1e-2, integralIntervs=4)
    assert api.dynamics().as_dict() == d
    assert api.dynamics(vmax=1.0).vmax == 1.0
    with pytest.raises(ValueError):
        api.dynamics(vmx=1.0)


def test_sampled_rates_match_the_polynomial():
    from implicit_svsdf_planner_b200 import plan

    rng = np.random.default_rng(2)
    T, b = random_traj(rng, 3, tmin=0.5, tmax=2.0)
    s, v, w = plan.sampled_rates(T, b, samples=11)
    c = b.reshape(3, 3, 6)
    for i in range(3):
        for m in range(11):
            t = s[i, m]
            vel = [sum(k * c[dd, i, k] * t ** (k - 1) for k in range(1, 6)) for dd in range(3)]
            assert abs(v[i, m] - math.hypot(vel[0], vel[1])) <= 1e-12 * (1 + abs(v[i, m]))
            assert abs(w[i, m] - vel[2]) <= 1e-12 * (1 + abs(w[i, m]))
    assert s[:, 0].tolist() == [0.0] * 3 and np.allclose(s[:, -1], T)
    rep = plan.dynamics_report(dict(vmax=1e9, omgmax=1e9), T, b)
    assert rep["within_limits"] and rep["v_peak"] == v.max() and rep["omg_peak"] == np.abs(w).max()
