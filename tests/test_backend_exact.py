"""CPU: the back end's arithmetic against the mathematics it computes, at 60 significant digits (mpmath).

The reference here is written from the definitions, not from csrc/host/minco.hpp's formulas:
  - MINCO: the minimum-jerk spline through the waypoints is the solution of the 6N linear conditions (head and tail position, velocity
    and acceleration; each waypoint reached by the piece that ends there and the piece that starts there; velocity to snap continuous
    across every waypoint).  They are written here in their own order and solved by Gaussian elimination with partial pivoting at 60
    digits.  The energy is the integral of |c'''(t)|^2 over each piece, integrated as a polynomial; dE/dc and dE/dT are the exact
    derivatives of that integral (dE/dT_i = |c_i'''(T_i)|^2).
  - The adjoint (svsdf_minco_propagate) of phi(q, T) = sum W . c(q, T) + wT . T: lambda = A^-T W at 60 digits, d phi / d q = lambda at
    the two rows where q enters, d phi / d T_i = wT_i - lambda^T (dA / dT_i) c; a few entries are checked against mp.diff of phi.
  - The tau maps: T = tau^2 / 2 + tau + 1 (tau > 0), 1 / (tau^2 / 2 - tau + 1) (tau <= 0), and their inverses.
  - The dynamics penalty: the trapezoid-sampled cost of host::dynamics_penalty's docstring evaluated at 60 digits; gradC and gradT are
    mp.diff derivatives of that sampled cost, not its hand-written chain rule.

Bounds are c * u * M, u = 2^-53, with M a condition measure stated at each check and c set from the largest ratio observed over all
cases (recorded next to each constant).  The product's MINCO eliminates without pivoting, as the reference's minco.hpp does: where the
durations span four to five decades that costs accuracy no condition measure of the system accounts for (see CONTRAST below).
backwardGradT (the tau map's chain rule) has no host entry and is not compared with exact values here; the bit-for-bit tests of
test_gpu_backend_edges.py pin the device's to the host's.
"""
import math

import mpmath as mp
import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api

DPS = 60
U = 2.0 ** -53

# ---------------------------------------------------------------------------------------------------------------------------------------
# the cases: head / tail states with large velocities and accelerations, durations at their limits


def _state(rng, v, a):
    s = np.zeros((3, 3))
    s[:, 0] = rng.uniform(-5, 5, 3)
    s[:, 1] = rng.normal(0, v, 3)
    s[:, 2] = rng.normal(0, a, 3)
    return s


def make_case(N, T, seed, v=8.0, a=40.0):
    """(init_s, final_s, q (3 x N-1), T): waypoints a seeded walk whose steps scale with the durations."""
    rng = np.random.default_rng(seed)
    T = np.asarray(T, dtype=np.float64)
    init_s, final_s = _state(rng, v, a), _state(rng, v, a)
    steps = rng.normal(0.0, 1.0, (3, N)) * np.minimum(T, 5.0)
    q = init_s[:, :1] + np.cumsum(steps, axis=1)[:, : N - 1]
    final_s[:, 0] = q[:, -1] + steps[:, -1] if N > 1 else final_s[:, 0]
    return init_s, final_s, q, T


def _durations(name, N, rng):
    if name == "typical":
        return rng.uniform(0.8, 2.5, N)
    if name == "1ms_among_2s":
        T = np.full(N, 2.0)
        T[N // 2] = 1e-3
        return T
    if name == "loguniform":
        T = np.exp(rng.uniform(math.log(1e-3), math.log(10.0), N))
        T[0], T[-1] = 1e-3, 10.0
        return T
    if name == "D299.9":
        T = rng.uniform(0.5, 1.5, N)
        return T * (299.9 / T.sum())
    if name == "250s":
        T = np.full(N, 2.0)
        T[1] = 250.0
        return T
    raise KeyError(name)


# (name, N, durations): N = 1 is refused by the host MINCO (svsdf_minco_forward needs a waypoint-free N >= 2)
CASES = ([(f"typical_N{N}", N, "typical") for N in (2, 32, 33, 64)]
         + [("1ms_among_2s_N8", 8, "1ms_among_2s"), ("1ms_among_2s_N33", 33, "1ms_among_2s"), ("loguniform_N16", 16, "loguniform"),
            ("loguniform_N64", 64, "loguniform"), ("D299.9_N64", 64, "D299.9"), ("250s_N2", 2, "250s"), ("250s_N4", 4, "250s")])


def case(name):
    for k, (nm, N, kind) in enumerate(CASES):
        if nm == name:
            rng = np.random.default_rng(1000 + k)
            return make_case(N, _durations(kind, N, rng), 2000 + k)
    raise KeyError(name)


# ---------------------------------------------------------------------------------------------------------------------------------------
# 60-digit linear algebra


def gauss(rows, rhs, n):
    """Solve sum_c rows[r][c] x[c] = rhs[r][m] (m right-hand sides) by Gaussian elimination with partial pivoting; rows are dicts
    column -> mpf (zeros omitted).  Returns x as a list of n lists of m values."""
    rows = [dict(r) for r in rows]
    rhs = [list(b) for b in rhs]
    m = len(rhs[0])
    free = set(range(n))
    order = []
    for col in range(n):
        cand = [r for r in free if rows[r].get(col, 0) != 0]
        p = max(cand, key=lambda r: abs(rows[r][col]))
        free.discard(p)
        order.append(p)
        prow, pv = rows[p], rows[p][col]
        for r in cand:
            if r == p:
                continue
            f = rows[r].pop(col) / pv
            for c, v in prow.items():
                if c != col:
                    rows[r][c] = rows[r].get(c, 0) - f * v
            for k in range(m):
                rhs[r][k] -= f * rhs[p][k]
    x = [[mp.mpf(0)] * m for _ in range(n)]
    for col in range(n - 1, -1, -1):
        p = order[col]
        for k in range(m):
            s = rhs[p][k]
            for c, v in rows[p].items():
                if c != col:
                    s -= v * x[c][k]
            x[col][k] = s / rows[p][col]
    return x


def _deriv_row(m, t, i):
    """d^m/dt^m of piece i's polynomial at t: {6 i + k: k! / (k - m)! t^(k - m)}, and its derivative with respect to t."""
    row, drow = {}, {}
    for k in range(m, 6):
        f = math.factorial(k) // math.factorial(k - m)
        row[6 * i + k] = f * t ** (k - m)
        if k > m:
            drow[6 * i + k] = f * (k - m) * t ** (k - m - 1)
    return row, drow


def _mpf(x):
    return x if isinstance(x, mp.mpf) else mp.mpf(float(x))


def _neg(row):
    return {c: -v for c, v in row.items()}


class Minco:
    """The 6N conditions of the minimum-jerk spline at 60 digits.  self.rows (dicts), self.rhs (6N x 3), self.dT[r] = (i, d row / d T_i)
    for the rows that depend on a duration, self.qrows[i] = the two rows whose right-hand side is waypoint i."""

    def __init__(self, init_s, final_s, q, T):
        with mp.workdps(max(DPS, mp.mp.dps)):
            N = len(T)
            self.N, self.n = N, 6 * N
            self.T = [t if isinstance(t, mp.mpf) else mp.mpf(float(t)) for t in T]
            rows, rhs, dT, qrows = [], [], {}, []
            z3 = [mp.mpf(0)] * 3
            for i in range(N - 1):  # waypoint i: reached at the end of piece i and at the start of piece i + 1
                qi = [q[d][i] if isinstance(q[d][i], mp.mpf) else mp.mpf(float(q[d][i])) for d in range(3)]
                r, dr = _deriv_row(0, self.T[i], i)
                dT[len(rows)] = (i, dr)
                rows.append(r); rhs.append(qi)
                rows.append(_deriv_row(0, mp.mpf(0), i + 1)[0]); rhs.append(qi)
                qrows.append((len(rows) - 2, len(rows) - 1))
            for i in range(N - 1):  # velocity, acceleration, jerk and snap continuous across waypoint i
                for m in range(1, 5):
                    r, dr = _deriv_row(m, self.T[i], i)
                    r.update(_neg(_deriv_row(m, mp.mpf(0), i + 1)[0]))
                    dT[len(rows)] = (i, dr)
                    rows.append(r); rhs.append(z3)
            for m in range(3):  # head and tail
                rows.append(_deriv_row(m, mp.mpf(0), 0)[0]); rhs.append([mp.mpf(float(init_s[d, m])) for d in range(3)])
                r, dr = _deriv_row(m, self.T[N - 1], N - 1)
                dT[len(rows)] = (N - 1, dr)
                rows.append(r); rhs.append([mp.mpf(float(final_s[d, m])) for d in range(3)])
            assert len(rows) == self.n
            self.rows, self.rhs, self.dT, self.qrows = rows, rhs, dT, qrows
            self.c = gauss(rows, rhs, self.n)  # c[6 i + k][d]

    def coeffs(self):
        """6N x 3 float64 view of the exact coefficients (for condition measures)"""
        return np.array([[float(v) for v in r] for r in self.c])

    def adjoint(self, W, wT):
        """exact gradient of phi = sum W . c + wT . T: (gradQ 3 x (N-1), gradT N) as mpf, and lambda"""
        with mp.workdps(max(DPS, mp.mp.dps)):
            n = self.n
            cols = [dict() for _ in range(n)]
            for r, row in enumerate(self.rows):
                for c, v in row.items():
                    cols[c][r] = v
            lam = gauss(cols, [[_mpf(W[r][d]) for d in range(3)] for r in range(n)], n)
            gq = [[lam[a][d] + lam[b][d] for a, b in self.qrows] for d in range(3)]
            gT = [_mpf(w) for w in wT]
            for r, (i, dr) in self.dT.items():
                for d in range(3):
                    gT[i] -= lam[r][d] * sum(v * self.c[c][d] for c, v in dr.items())
            return gq, gT, lam


def dense(mc):
    """float64 A of the conditions, and |A^-1| from an equilibrated inverse (columns scaled by the piece's T^k, rows by their max)"""
    n = mc.n
    A = np.zeros((n, n))
    for r, row in enumerate(mc.rows):
        for c, v in row.items():
            A[r, c] = float(v)
    T = np.array([float(t) for t in mc.T])
    cs = np.array([T[c // 6] ** (c % 6) for c in range(n)])
    As = A * cs[None, :]
    rs = 1.0 / np.abs(As).max(axis=1)
    inv = np.linalg.inv(As * rs[:, None])  # (R A C)^-1 = C^-1 A^-1 R^-1
    Ainv_abs = np.abs(inv) * cs[:, None] * rs[None, :]
    return A, Ainv_abs


# ---------------------------------------------------------------------------------------------------------------------------------------
# energy as an integral


def _jerk_poly(cp, a, b):
    """c'''(t) = sum_j p_j t^j of one piece / dimension from coefficients cp (6)"""
    return [6 * cp[3], 24 * cp[4], 60 * cp[5]]


def _polymul(p, q):
    out = [0] * (len(p) + len(q) - 1)
    for i, a in enumerate(p):
        for j, b in enumerate(q):
            out[i + j] += a * b
    return out


def _integral(p, T):
    return sum(a * T ** (j + 1) / (j + 1) for j, a in enumerate(p))


def _peval(p, t):
    return sum(a * t ** j for j, a in enumerate(p))


def energy_exact(c, T, absolute=False):
    """E = sum_i int_0^T_i |c_i'''|^2, dE/dc (6N x 3), dE/dT (N) at coefficients c[6 i + k][d] (any numbers), at 60 digits.  With
    absolute=True the same with |c| (the sum of the magnitudes of every term: the condition measure of a floating-point evaluation)."""
    with mp.workdps(max(DPS, mp.mp.dps)):
        N = len(T)
        E, gC, gT = mp.mpf(0), [[mp.mpf(0)] * 3 for _ in range(6 * N)], []
        for i in range(N):
            Ti = mp.mpf(float(T[i]))
            gti = mp.mpf(0)
            for d in range(3):
                cp = [mp.mpf(float(c[6 * i + k][d])) if not isinstance(c[6 * i + k][d], mp.mpf) else c[6 * i + k][d] for k in range(6)]
                if absolute:
                    cp = [abs(v) for v in cp]
                j = _jerk_poly(cp, 0, 0)
                E += _integral(_polymul(j, j), Ti)
                gti += _peval(j, Ti) ** 2
                for k in (3, 4, 5):  # d/dc_k int j^2 = int 2 j (d j / d c_k),  d j / d c_k = k (k-1) (k-2) t^(k-3)
                    dj = [0] * (k - 3) + [k * (k - 1) * (k - 2)]
                    gC[6 * i + k][d] = 2 * _integral(_polymul(j, dj), Ti)
            gT.append(gti)
        return E, gC, gT


# ---------------------------------------------------------------------------------------------------------------------------------------
# MINCO forward and adjoint


def piece_norms(x, N):
    """per piece 2-norm of a 6N x 3 array"""
    return np.sqrt((np.asarray(x, dtype=np.float64).reshape(N, 6, 3) ** 2).sum(axis=(1, 2)))


def _err(host, exact):
    """host - exact elementwise at 60 digits, as float64"""
    with mp.workdps(max(DPS, mp.mp.dps)):
        return np.array([float(mp.mpf(float(h)) - e) for h, e in zip(np.ravel(host), exact)])


def coeff_measure(mc, Ainv_abs, A):
    """Skeel's measure |A^-1| (|A| |c| + |b|), 6N x 3: first-order bound / u of a componentwise backward-stable solve"""
    c = np.abs(mc.coeffs())
    b = np.abs(np.array([[float(v) for v in r] for r in mc.rhs]))
    return Ainv_abs @ (np.abs(A) @ c + b)


# Observed maxima of error / (u M) over CASES; each constant allows a few times that.
#   coefficients, per piece (Skeel's measure):          2.7 (D299.9_N64)          -> C_COEF = 16
#   energy:                                             0.79                      -> C_E = 8
#   dE/dc per piece, dE/dT per piece:                   1.5, 2.9 (loguniform_N16) -> C_DE = 16
#   adjoint gradQ per waypoint:                         2.9 (D299.9_N64)          -> C_ADJ_Q = 16
#   adjoint gradT per piece:                            0.25 (1ms_among_2s_N33)   -> C_ADJ_T = 1
# Elimination without pivoting.  The product's MINCO factorises the 6N system without pivoting and reuses that LU for the adjoint's
# transposed solve, as the reference's MINCO_S3NU does; test_unpivoted_cases_are_the_references_bits checks that the reference gives
# the same coefficients and gradQ, bit for bit, on these cases.  Where it shows growth no condition measure of the system accounts for:
#   CONTRAST (durations spanning four to five decades): coefficients 22 / 77 / 4075 and gradT 7.4 / 5430 / 1650 (loguniform_N16 /
#     loguniform_N64 / 250s_N4).  On 250s_N4 the worst piece (a 2 s piece after the 250 s one) is off by 2e-11 relative, where LAPACK's
#     pivoted solve of the same float64 system gets that piece within 6e-16.  The device back end (test_gpu_backend_edges.py) reaches
#     14 600 on 250s_N4 (its durations come through backward_T / forward_T, one ulp away): C_CONTRAST = 2^16.
#   ADJ_GROWTH, gradQ per waypoint: CONTRAST and a 1 ms piece among 2 s pieces: 132 / 47 (1ms_among_2s_N8 / N33, where a pivoted
#     float64 solve stays within 0.3 / 0.5), 227 / 1720 (loguniform_N16 / 250s_N4): C_CONTRAST.  loguniform_N64 reaches 9.4e5 (2e-8
#     relative at one waypoint, 1.5e5 times a pivoted solve's error there; the pivoted solve itself exceeds this float64-computed measure
#     by 8e5 on another waypoint): C_ADJ_LOG64 = 2^22.
C_COEF, C_E, C_DE, C_ADJ_Q, C_ADJ_T, C_CONTRAST, C_ADJ_LOG64 = 16.0, 8.0, 16.0, 16.0, 1.0, 65536.0, 4194304.0
CONTRAST = {"loguniform_N16", "loguniform_N64", "250s_N4"}
ADJ_GROWTH = CONTRAST | {"1ms_among_2s_N8", "1ms_among_2s_N33"}


@pytest.fixture(scope="module")
def exact_cases():
    out = {}
    for name, N, _ in CASES:
        init_s, final_s, q, T = case(name)
        mc = Minco(init_s, final_s, q, T)
        A, Ainv_abs = dense(mc)
        out[name] = (init_s, final_s, q, T, mc, A, Ainv_abs)
    return out


def _ratio(err, meas):
    return float(np.max(err / (U * np.maximum(meas, 1e-300))))


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_minco_forward_is_the_exact_spline(exact_cases, name):
    """Coefficients per piece within C_COEF u Skeel; energy and its partials (at the product's own coefficients) within c u sum|terms|."""
    init_s, final_s, q, T, mc, A, Ainv_abs = exact_cases[name]
    N = len(T)
    b, e, gc, gt = api.minco_forward(init_s, final_s, q, T)
    flat = [v for r in mc.c for v in r]
    err = _err(b, flat).reshape(6 * N, 3)
    r_coef = _ratio(piece_norms(err, N), piece_norms(coeff_measure(mc, Ainv_abs, A), N))
    assert r_coef <= (C_CONTRAST if name in CONTRAST else C_COEF), (name, r_coef)
    # the energy and its partials of the product's coefficients
    cm = [[mp.mpf(float(v)) for v in row] for row in b]
    E, gC, gT = energy_exact(cm, T)
    Ea, gCa, gTa = energy_exact(cm, T, absolute=True)
    r_e = abs(float(mp.mpf(e) - E)) / (U * float(Ea))
    assert r_e <= C_E, (name, r_e)
    errc = _err(gc, [v for r in gC for v in r]).reshape(6 * N, 3)
    measc = np.array([[float(v) for v in r] for r in gCa])
    r_c = _ratio(piece_norms(errc, N), piece_norms(measc, N))
    errt = np.abs(_err(gt, gT))
    r_t = _ratio(errt, np.array([float(v) for v in gTa]))
    assert r_c <= C_DE and r_t <= C_DE, (name, r_c, r_t)
    print(f"{name}: coef {r_coef:.3g} E {r_e:.3g} dE/dc {r_c:.3g} dE/dT {r_t:.3g}")


def adjoint_measures(mc, A, Ainv_abs, lam):
    """first-order error measures / u of the adjoint: gradQ (3 x (N-1)), gradT (N)"""
    N = mc.N
    L = np.abs(np.array([[float(v) for v in r] for r in lam]))
    W = np.abs(np.array([[float(v) for v in r] for r in mc._W]))
    Sl = Ainv_abs.T @ (np.abs(A).T @ L + W)
    Sc = coeff_measure(mc, Ainv_abs, A)
    c = np.abs(mc.coeffs())
    mq = np.array([[Sl[a, d] + Sl[b, d] for a, b in mc.qrows] for d in range(3)])
    mt = np.abs(np.asarray(mc._wT, dtype=np.float64)).copy()
    for r, (i, dr) in mc.dT.items():
        for d in range(3):
            for col, v in dr.items():
                v = abs(float(v))
                mt[i] += (L[r, d] + Sl[r, d]) * v * c[col, d] + L[r, d] * v * Sc[col, d]
    return mq, mt


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_minco_adjoint_is_the_exact_gradient(exact_cases, name):
    """svsdf_minco_propagate(W, wT) = the gradient of phi = sum W . c(q, T) + wT . T: per waypoint and per piece within c u M."""
    init_s, final_s, q, T, mc, A, Ainv_abs = exact_cases[name]
    N = len(T)
    mc._W, mc._wT = adjoint_weights(N)
    gq, gT = api.minco_propagate(init_s, final_s, q, T, mc._W, mc._wT)
    xq, xT, lam = mc.adjoint(mc._W, mc._wT)
    mq, mt = adjoint_measures(mc, A, Ainv_abs, lam)
    eq = _err(gq, [v for r in xq for v in r]).reshape(3, N - 1)
    et = np.abs(_err(gT, xT))
    # every waypoint's gradQ (2-norm over x, y, yaw) and every piece's gradT against its own measure
    r_q = _ratio(np.sqrt((eq ** 2).sum(axis=0)), np.sqrt((mq ** 2).sum(axis=0)))
    r_t = _ratio(et, mt)
    print(f"{name}: gradQ {r_q:.3g} gradT {r_t:.3g}")
    assert r_q <= (C_ADJ_LOG64 if name == "loguniform_N64" else C_CONTRAST if name in ADJ_GROWTH else C_ADJ_Q), (name, r_q)
    assert r_t <= (C_CONTRAST if name in CONTRAST else C_ADJ_T), (name, r_t)


def adjoint_weights(N):
    rng = np.random.default_rng(N + 7)
    return rng.normal(size=(6 * N, 3)), rng.normal(size=N)


@pytest.mark.parametrize("name", sorted(ADJ_GROWTH))
def test_unpivoted_cases_are_the_references_bits(name):
    """The cases whose bounds allow for the elimination's growth: the reference's own MINCO_S3NU (compiled from its source into
    oracle/_ref where the reference tree exists) gives the product's coefficients and gradQ bit for bit, so the growth is the
    reference's arithmetic and not a slip of the restatement."""
    from oracle import ref_py
    if not ref_py.available("glibc"):
        pytest.skip("oracle/_ref not built (the reference tree is absent)")
    init_s, final_s, q, T = case(name)
    N = len(T)
    r = ref_py.RefPath("star")
    r.set_conditions(init_s, final_s, N)
    rb, _, _, _ = r.minco_forward(q, T)
    b, *_ = api.minco_forward(init_s, final_s, q, T)
    assert np.array_equal(np.ascontiguousarray(b.T).reshape(-1).view(np.uint64), rb.view(np.uint64)), name
    W, wT = adjoint_weights(N)
    rq, _ = r.minco_propagate(np.ascontiguousarray(W.T).reshape(-1), wT)
    gq, _ = api.minco_propagate(init_s, final_s, q, T, W, wT)
    assert np.array_equal(gq.view(np.uint64), rq.view(np.uint64)), name


def test_adjoint_reference_is_the_derivative_of_phi():
    """The 60-digit adjoint itself against mp.diff of phi(q, T) (a fresh 60-digit solve per evaluation) on a few entries."""
    for name in ("typical_N2", "1ms_among_2s_N8"):
        init_s, final_s, q, T = case(name)
        N = len(T)
        rng = np.random.default_rng(5)
        W, wT = rng.normal(size=(6 * N, 3)), rng.normal(size=N)
        xq, xT, _ = Minco(init_s, final_s, q, T).adjoint(W, wT)
        with mp.workdps(max(DPS, mp.mp.dps)):
            qm = [[mp.mpf(float(q[d, i])) for i in range(N - 1)] for d in range(3)]
            Tm = [mp.mpf(float(t)) for t in T]

            def phi(qq, TT):
                c = Minco(init_s, final_s, qq, TT).c
                return sum(mp.mpf(float(W[r, d])) * c[r][d] for r in range(6 * N) for d in range(3)) + sum(
                    mp.mpf(float(w)) * t for w, t in zip(wT, TT))

            for i in sorted({0, N // 2, N - 1}):
                fd = mp.diff(lambda t: phi(qm, Tm[:i] + [t] + Tm[i + 1:]), Tm[i])
                assert abs(fd - xT[i]) <= mp.mpf(10) ** -25 * (1 + abs(xT[i])), (name, i)
            for d, i in ((0, 0), (2, N - 2)):
                def f(v, d=d, i=i):
                    qq = [list(r) for r in qm]
                    qq[d][i] = v
                    return phi(qq, Tm)
                fd = mp.diff(f, qm[d][i])
                assert abs(fd - xq[d][i]) <= mp.mpf(10) ** -25 * (1 + abs(xq[d][i])), (name, d, i)


# ---------------------------------------------------------------------------------------------------------------------------------------
# tau maps


def forward_T_exact(tau):
    t = mp.mpf(float(tau))
    return t * t / 2 + t + 1 if tau > 0 else 1 / (t * t / 2 - t + 1)


def tau_sweep():
    t = np.r_[np.linspace(-1e3, 1e3, 4001), np.logspace(-300, 3, 607), -np.logspace(-300, 3, 607), 0.0, -0.0, 1e-300, -1e-300,
              5e-324, -5e-324, np.nextafter(0.0, 1.0) * 3, 1e3, -1e3]
    return t


def test_forward_T_is_within_four_ulps():
    """T(tau) over tau in +-1e3, +-0, +-1e-300, subnormals and the branch switch at 0 (tau = +-0 and tiny tau give T = 1).  Observed
    maximum: 2.1 ulps (three roundings on the positive branch, four on the other)."""
    tau = tau_sweep()
    T = api.forward_T(tau)
    with mp.workdps(DPS):
        err = np.array([float(abs(mp.mpf(float(h)) - forward_T_exact(t))) for h, t in zip(T, tau)])
        ex = np.array([float(forward_T_exact(t)) for t in tau])
    ulps = err / np.spacing(ex)
    assert ulps.max() <= 4.0, (ulps.max(), tau[ulps.argmax()])
    assert (T[tau == 0.0] == 1.0).all()
    print(f"forward_T: max {ulps.max():.3g} ulps")


def test_backward_T_is_within_two_ulps_of_its_terms():
    """tau(T) = sqrt(2T - 1) - 1 (T > 1), 1 - sqrt(2 / T - 1) (T <= 1): T = 1 and 1 +- 1 ulp, near 300 s, 1e-3 and the sweep's T.  The
    difference cancels next to T = 1, so the bound is on the scale of its terms (2 ulps of sqrt(.) + 1, observed 0.74): relative to tau
    itself, tau(1 + k ulp) is off by up to ~2^51 / k ulps, in the reference's formula as here."""
    T = np.r_[1.0, np.nextafter(1.0, 2.0), np.nextafter(1.0, 0.0), 1.0 + 2 ** -30, 1.0 - 2 ** -30, 299.9, np.nextafter(300.0, 0.0), 300.0,
              1e-3, 250.0, 5e5, 1e-6, api.forward_T(tau_sweep()[::7])]
    T = T[T > 0]
    tau = api.backward_T(T)
    worst = 0.0
    with mp.workdps(DPS):
        for h, t in zip(tau, T):
            tm = mp.mpf(float(t))
            sq = mp.sqrt(2 * tm - 1) if t > 1.0 else mp.sqrt(2 / tm - 1)
            ex = sq - 1 if t > 1.0 else 1 - sq
            err = float(abs(mp.mpf(float(h)) - ex))
            worst = max(worst, err / np.spacing(float(sq + 1)))
            assert err <= 2.0 * np.spacing(float(sq + 1)), (t, h, float(ex))
            if t == 1.0:
                assert h == 0.0
    print(f"backward_T: max {worst:.3g} ulps of its terms")
    # round trip at the ends of the range the back end uses
    for t in (1e-3, 299.9, 250.0, 1.0):
        assert abs(api.forward_T(api.backward_T(np.array([t])))[0] - t) <= 8 * np.spacing(t) * max(1.0, t)


# ---------------------------------------------------------------------------------------------------------------------------------------
# the dynamics penalty


def _sl1(x, mu):
    """smoothed L1 at 60 digits: 0 below 0 (the sample adds nothing), the cubic on [0, mu], x - mu / 2 above"""
    if x < 0:
        return mp.mpf(0)
    if x > mu:
        return x - mu / 2
    return (mu - x / 2) * (x / mu) ** 3


def dyn_piece_cost(d, Ti, cp):
    """the trapezoid-sampled penalty of one piece: sum_j node_j (T_i / res) (w_v sl1(|v_xy|^2 - vmax^2) + w_omg sl1(v_yaw^2 - omgmax^2))
    at s_j = j T_i / res, node = 1/2 at j = 0 and j = res; cp[dim][k] the piece's coefficients"""
    res = d["integralIntervs"]
    mu = mp.mpf(d["smoothingEps"])
    vs, os_ = mp.mpf(d["vmax"]) ** 2, mp.mpf(d["omgmax"]) ** 2
    step = Ti / res
    tot = mp.mpf(0)
    for j in range(res + 1):
        s = j * step
        vel = [sum(k * cp[dd][k] * s ** (k - 1) for k in range(1, 6)) for dd in range(3)]
        pena = mp.mpf(d["weight_v"]) * _sl1(vel[0] ** 2 + vel[1] ** 2 - vs, mu) + mp.mpf(d["weight_omg"]) * _sl1(vel[2] ** 2 - os_, mu)
        tot += (mp.mpf(1) / 2 if j in (0, res) else 1) * step * pena
    return tot


def dyn_exact(d, T, b):
    """(cost, gradT, gradC 18N column-major) at 60 digits: the sampled cost and its mp.diff derivatives"""
    N = len(T)
    n = 6 * N
    with mp.workdps(DPS):
        cost, gT, gC = mp.mpf(0), [], [mp.mpf(0)] * (18 * N)
        for i in range(N):
            Ti = mp.mpf(float(T[i]))
            cp = [[mp.mpf(float(b[dd * n + 6 * i + k])) for k in range(6)] for dd in range(3)]
            cost += dyn_piece_cost(d, Ti, cp)
            gT.append(mp.diff(lambda t: dyn_piece_cost(d, t, cp), Ti))
            for dd in range(3):
                for k in range(1, 6):  # the penalty does not depend on c_0
                    def f(v, dd=dd, k=k):
                        cq = [list(r) for r in cp]
                        cq[dd][k] = v
                        return dyn_piece_cost(d, Ti, cq)
                    gC[dd * n + 6 * i + k] = mp.diff(f, cp[dd][k])
        return cost, gT, gC


def dyn_measures(d, T, b):
    """the magnitudes a float64 evaluation of the sampled cost and of its derivatives rounds, per quantity (cost, gradT, gradC): every
    term with |.|, the violations' rounding carried through df and ddf"""
    N = len(T)
    n = 6 * N
    res, mu = d["integralIntervs"], d["smoothingEps"]
    lims = (d["vmax"] ** 2, d["omgmax"] ** 2)
    ws = (d["weight_v"], d["weight_omg"])
    mc, mt, mg = 0.0, np.zeros(N), np.zeros(18 * N)
    for i in range(N):
        step = T[i] / res
        c = np.array([[b[dd * n + 6 * i + k] for k in range(6)] for dd in range(3)])
        for j in range(res + 1):
            s = j * step
            node, alpha = (0.5 if j in (0, res) else 1.0), j / res
            b1 = np.array([k * s ** (k - 1) if k else 0.0 for k in range(6)])
            b2 = np.array([k * (k - 1) * s ** (k - 2) if k > 1 else 0.0 for k in range(6)])
            vel, vabs, aabs = c @ b1, np.abs(c) @ np.abs(b1), np.abs(c) @ np.abs(b2)
            for dims, lim, w in (((0, 1), lims[0], ws[0]), ((2,), lims[1], ws[1])):
                x = sum(vel[k] ** 2 for k in dims) - lim
                vm = sum(vabs[k] ** 2 for k in dims) + lim
                if x < -1e-9 * vm:
                    continue
                x = max(x, 0.0)
                if x > mu:
                    f, df, ddf = x - 0.5 * mu, 1.0, 0.0
                else:
                    f, df, ddf = (mu - 0.5 * x) * (x / mu) ** 3, 3 * x * x / mu ** 2 - 2 * x ** 3 / mu ** 3, 6 * x / mu ** 2 - 6 * x * x / mu ** 3
                pm = w * (abs(f) + abs(df) * vm)
                mc += node * step * pm
                mt[i] += node * pm / res
                for k in dims:
                    gv = w * 2 * (abs(df) * vabs[k] + abs(ddf) * vm * abs(vel[k]))
                    mt[i] += gv * aabs[k] * alpha * node * step
                    mg[k * n + 6 * i: k * n + 6 * i + 6] += np.abs(b1) * gv * node * step
    return mc, mt, mg


def _dyn(**kw):
    d = dict(vmax=2.0, omgmax=1.0, weight_v=10.0, weight_omg=7.0, smoothingEps=0.5, integralIntervs=4)
    d.update(kw)
    return d


def _minco_traj(name):
    init_s, final_s, q, T = case(name)
    b, *_ = api.minco_forward(init_s, final_s, q, T)
    return T, np.ascontiguousarray(b.T).reshape(-1)


def _speeds(T, b, res):
    """median |v_xy| and |v_yaw| over the samples"""
    N = len(T)
    c = b.reshape(3, N, 6)
    v, w = [], []
    for i in range(N):
        for j in range(res + 1):
            s = j * T[i] / res
            vel = [sum(k * c[dd, i, k] * s ** (k - 1) for k in range(1, 6)) for dd in range(3)]
            v.append(math.hypot(vel[0], vel[1]))
            w.append(abs(vel[2]))
    return float(np.median(v)), float(np.median(w))


def _edge_piece():
    """two 1 s pieces; at s = 0 every velocity is the coefficient c_1 itself, so the violations there are exact"""
    b = np.zeros((3, 2, 6))
    b[:, 0, 1] = (3.0, 4.0, 0.0)    # |v| = 5 = vmax exactly: violation 0 (active, f = 0); yaw rate 0
    b[:, 1, 1] = (1.5, 0.0, 0.0)    # |v|^2 - 1 = 1.25 = mu (vmax = 1 for the second set of limits)
    b[:, 0, 2:] = [[0.4, -0.3, 0.1, 0.02], [-0.2, 0.1, 0.05, -0.01], [0.0, 0.0, 0.0, 0.0]]
    b[:, 1, 2:] = [[-0.5, 0.2, 0.0, 0.03], [0.3, -0.1, 0.02, 0.0], [0.0, 0.0, 0.0, 0.0]]
    return np.array([1.0, 1.0]), b.reshape(-1)


def dyn_cases():
    out = []
    for name, res in (("typical_N2", 1), ("typical_N2", 64), ("typical_N64", 4), ("1ms_among_2s_N8", 64), ("250s_N4", 16),
                      ("loguniform_N16", 8)):
        T, b = _minco_traj(name)
        v, w = _speeds(T, b, res)
        out.append((f"{name}_res{res}", T, b, _dyn(vmax=v, omgmax=w, smoothingEps=0.3 * v * v, integralIntervs=res)))
    T, b = _edge_piece()
    out.append(("violation_0", T, b, _dyn(vmax=5.0, omgmax=0.5, smoothingEps=0.25, integralIntervs=3)))
    for tag, mu in (("mu", 1.25), ("mu_minus", np.nextafter(1.25, 0.0)), ("mu_plus", np.nextafter(1.25, 2.0))):
        out.append((f"violation_{tag}", T, b, _dyn(vmax=1.0, omgmax=0.5, smoothingEps=mu, integralIntervs=2)))
    return out


# observed maxima of error / (u M): cost 0.14, gradT 0.66, gradC 2.6 (loguniform_N16_res8) -> C_DYN = 8
C_DYN = 8.0
DYN_CASES = dyn_cases()


@pytest.mark.parametrize("k", range(len(DYN_CASES)), ids=[c[0] for c in DYN_CASES])
def test_dynamics_penalty_is_the_sampled_cost_and_its_derivatives(k):
    """svsdf_dynamics_penalty against the 60-digit sampled cost; gradT and gradC against mp.diff of it.  Entry by entry within
    C_DYN u M, M every term's magnitude (dyn_measures)."""
    name, T, b, d = DYN_CASES[k]
    cost, gT, gC = api.dynamics_penalty(T, b, d)
    xc, xT, xC = dyn_exact(d, T, b)
    mc, mt, mg = dyn_measures(d, T, b)
    assert mc > 0, name  # some sample is active
    r_c = abs(float(mp.mpf(cost) - xc)) / (U * mc)
    r_t = _ratio(np.abs(_err(gT, xT)), mt)
    r_g = _ratio(np.abs(_err(gC, xC)), mg)
    print(f"{name}: cost {r_c:.3g} gradT {r_t:.3g} gradC {r_g:.3g}")
    assert r_c <= C_DYN and r_t <= C_DYN and r_g <= C_DYN, (name, r_c, r_t, r_g)
