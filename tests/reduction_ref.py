"""Restatement of the last stage of the cost path — the per-point penalty and chain rule (point_contribution,
csrc/svsdf_kernels.cuh) and the reduction of its terms into cost, gradC and gradT (outer_body's per-warp accumulators, the
interior slots of gsip_body, finalize_body) — in numpy, for the tests.

Every input of point_contribution is an output of svsdf_query: (px, py, sdf, t*, gx, gy), with the world-frame GSIP
direction at interior points.  The chain rule has no transcendental function except the pinned portable sin/cos
(oracle_py.sincos), so each term can be restated exactly:
  * point_terms: the per-point terms, operation by operation as point_contribution performs them.  Elementwise ufuncs only:
    numpy never contracts a * b + c, and every ufunc used here is correctly rounded.
  * exact_record: each output entry as the exactly rounded sum of its terms (math.fsum), with sum |terms|.
  * ordered_record: each output entry summed in the kernels' order (warp chains, CTA partials, the finalize lanes and
    shuffle tree, the interior slots, the gradT suffix).  Sums that must follow an order are explicit loops of `+` over
    columns; np.sum / np.add.reduce sum pairwise and are never used where the order matters.
  * gamma_bound: per entry the length h of the longest addition chain of that schedule and gamma_h * sum |terms|, the
    rigorous bound on |ordered - exact| for any summation order whose chains are at most h long.
Adding +0.0 to a sum that starts at +0.0 never changes it in round-to-nearest (the sum is never -0.0), so skipping a term
and adding a zero in its place give the same bits: the restatement pads with zeros where the kernels skip.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

U = 2.0 ** -53
WARPS_PER_CTA = 8   # kWarpsPerBlock
BATCHED_MIN = 16    # the runtime's rule: batched schedule when P >= 16 * grid * kWarpsPerBlock


def _sincos(x):
    from oracle import oracle_py

    return oracle_py.sincos(np.ascontiguousarray(x, dtype=np.float64))


def locate_piece(T, t):
    """Trajectory<5>::locatePieceIdx for an array of times: subtract durations while t > dur (strict), and past the last
    piece (idx == N) take the last piece with t += dur.  Returns (piece, local time)."""
    T = np.asarray(T, dtype=np.float64)
    t = np.array(t, dtype=np.float64, copy=True).reshape(-1)
    N = T.shape[0]
    piece = np.zeros(t.shape, dtype=np.int64)
    going = np.ones(t.shape, dtype=bool)
    for i in range(N):
        step = going & (t > T[i])
        t = np.where(step, t - T[i], t)
        piece += step
        going = step
    past = piece == N
    piece[past] = N - 1
    t = np.where(past, t + T[N - 1], t)
    return piece, t


def smoothed_l1(x, mu=0.01):
    """smoothedL1 (back_end_optimizer.hpp:316-340) elementwise: (ret, f, df); f = -1, df = 0 where it returns false."""
    x = np.asarray(x, dtype=np.float64)
    with np.errstate(all="ignore"):
        xdmu = x / mu
        sq = xdmu * xdmu
        mumxd2 = mu - 0.5 * x
        f_band = (mumxd2 * sq) * xdmu
        df_band = sq * ((-0.5) * xdmu + (3.0 * mumxd2) / mu)
    ret = ~(x < 0.0)
    hi = x > mu
    f = np.where(hi, x - 0.5 * mu, f_band)
    df = np.where(hi, 1.0, df_band)
    return ret, np.where(ret, f, -1.0), np.where(ret, df, 0.0)


def scale_inv(sched, t):
    """scale_inv (svsdf_kernels.cuh): the diagonal (ix, iy) of St^-1 by Eigen's size-3 cofactor formula, sin(w t + phi)."""
    a, b, w, phi = (np.asarray(sched[k], dtype=np.float64) for k in ("a", "b", "w", "phi"))
    s0, _ = _sincos(w[0] * t + phi[0])
    s1, _ = _sincos(w[1] * t + phi[1])
    sx = a[0] + s0 * b[0]
    sy = a[1] + s1 * b[1]
    inv = 1.0 / (sy * sx)
    return sy * inv, sx * inv


@dataclass
class Terms:
    """Per-point terms of the penalty.  gc[k, d, q] = beta_q * G_d (18 gradC terms), gdT, pena; zero where not active."""
    piece: np.ndarray     # [P] int
    s1: np.ndarray        # [P] local time at t*
    G: np.ndarray         # [P, 3]
    gc: np.ndarray        # [P, 3, 6]
    gdT: np.ndarray       # [P]
    pena: np.ndarray      # [P]
    active: np.ndarray    # [P] bool
    B: np.ndarray         # [P, 20]: magnitude bounds of pena, the 18 gc terms ([d][q]) and gdT (absolute values, see magnitudes)
    N: int


def _bases(s1):
    s2 = s1 * s1
    s3 = s2 * s1
    s4 = s2 * s2
    s5 = s4 * s1
    one = np.ones_like(s1)
    b0 = np.stack([one, s1, s2, s3, s4, s5], axis=1)
    b1 = np.stack([np.zeros_like(s1), one, 2.0 * s1, 3.0 * s2, 4.0 * s3, 5.0 * s4], axis=1)
    return b0, b1


def point_terms(pts, T, coeffs, sdf, tstar, g, weight_p, safety_hor, scale=None, rotate_interior=True):
    """point_contribution for every point.  pts [P, >= 2]; coeffs: MINCO b column-major (d * 6N + 6i + q); sdf, tstar [P];
    g [P, >= 2]: the gradient svsdf_query returns (body frame outside, world-frame GSIP direction inside: rotated to the body
    frame where sdf < 0 when rotate_interior; the oracle's per-point record is already rotated).  scale: None (rigid) or a
    dict a, b, w, phi of the deformable robot's schedule (point_contribution<SCALED>)."""
    pts = np.atleast_2d(np.asarray(pts, dtype=np.float64))
    T = np.asarray(T, dtype=np.float64).reshape(-1)
    N = T.shape[0]
    co = np.asarray(coeffs, dtype=np.float64).reshape(3, N, 6)  # [d][i][q]
    sdf = np.asarray(sdf, dtype=np.float64).reshape(-1)
    tstar = np.asarray(tstar, dtype=np.float64).reshape(-1)
    g = np.atleast_2d(np.asarray(g, dtype=np.float64))
    px, py = pts[:, 0].copy(), pts[:, 1].copy()
    gx, gy = g[:, 0].copy(), g[:, 1].copy()
    piece, s1 = locate_piece(T, tstar)
    b0, b1 = _bases(s1)
    c = co[:, piece, :]  # [3, P, 6]
    pos, vel = [], []
    for d in range(3):  # from 0.0 in ascending powers, one rounding per operation
        a = np.zeros_like(s1)
        v = np.zeros_like(s1)
        for q in range(6):
            a = a + c[d, :, q] * b0[:, q]
            v = v + c[d, :, q] * b1[:, q]
        pos.append(a)
        vel.append(v)
    sy, cy = _sincos(pos[2])
    if rotate_interior:  # :832 world -> body
        rot = sdf < 0
        g0 = cy * gx + sy * gy
        g1 = -sy * gx + cy * gy
        gx, gy = np.where(rot, g0, gx), np.where(rot, g1, gy)
    _, f, df = smoothed_l1(safety_hor - sdf, 0.01)
    active = f > 0
    if scale is None:
        ix = iy = None
        rg0 = -(cy * gx + (-sy) * gy)
        rg1 = -(sy * gx + cy * gy)
    else:
        ix, iy = scale_inv(scale, tstar)
        rg0 = -((ix * cy) * gx + (-(ix * sy)) * gy)
        rg1 = -((iy * sy) * gx + (iy * cy) * gy)
    sg0, sg1 = -df * rg0, -df * rg1
    d0, d1 = px - pos[0], py - pos[1]
    w0 = -sy * d0 + cy * d1
    w1 = -cy * d0 + -sy * d1
    gyaw = (-df * gx) * w0 + (-df * gy) * w1
    G = np.stack([weight_p * sg0, weight_p * sg1, weight_p * gyaw], axis=1)
    pena = weight_p * f
    gdT = -(G[:, 0] * vel[0] + G[:, 1] * vel[1] + G[:, 2] * vel[2])
    zero = ~active
    G[zero] = 0.0
    pena = np.where(active, pena, 0.0)
    gdT = np.where(active, gdT, 0.0)
    gc = b0[:, None, :] * G[:, :, None]  # beta_q * G_d (beta_0 = 1.0: G itself)
    B = magnitudes(c, b0, b1, d0, d1, gx, gy, f, weight_p, tstar, scale, ix, iy, safety_hor - sdf)
    B[zero] = 0.0
    return Terms(piece, s1, G, gc, gdT, pena, active, B, N)


def magnitudes(c, b0, b1, d0, d1, gx, gy, f, weight_p, tstar, scale, ix, iy, x):
    """B[k]: a bound on the magnitudes that enter each term of point k, from the same formulas on absolute values.  It is
    the scale of the difference between two evaluations of a term that round differently (contraction into FMAs):
    pos / vel carry the sums of |c_q beta_q|; sin and cos of a yaw known to within e carry 1 + |yaw| (their error is
    about e plus a few ulp); the scale's sine likewise carries 1 + |w t + phi|.  The FMA build's allowance is KAPPA * u * B
    (tests/test_gpu_reduction.py)."""
    with np.errstate(all="ignore"):
        pabs = [np.abs(c[d] * b0).sum(axis=1) for d in range(3)]  # order is irrelevant for a bound
        vabs = [np.abs(c[d] * b1).sum(axis=1) for d in range(3)]
        sc = 1.0 + pabs[2]  # sin / cos of yaw: |error| <~ (rounding of yaw) + ulps
        ga = np.abs(gx) + np.abs(gy)
        if scale is not None:
            a, b, w, phi = (np.asarray(scale[k], dtype=np.float64) for k in ("a", "b", "w", "phi"))
            arg = 1.0 + np.maximum(np.abs(w[0] * tstar) + abs(phi[0]), np.abs(w[1] * tstar) + abs(phi[1]))
            ib = np.maximum(np.abs(ix), np.abs(iy)) * (1.0 + np.max(np.abs(b) / (a - np.abs(b))) * arg)
        else:
            ib = 1.0
        dfa = np.where(x > 0.01, 1.0, 4.0)  # |df| and the terms of its band formula: sq (0.5 x / mu + 3 (mu - x / 2) / mu) <= 3.5
        gxy = weight_p * dfa * ib * ga * sc
        dist = np.abs(d0) + np.abs(d1) + pabs[0] + pabs[1]  # p - pos, pos known to within its rounding
        gyw = weight_p * dfa * ga * dist * sc
        Gb = np.stack([gxy, gxy, gyw], axis=1)
        B = np.zeros((len(x), 20))
        B[:, 0] = weight_p * (np.abs(f) + np.abs(x) + 0.01)
        B[:, 1:19] = (np.abs(b0)[:, None, :] * Gb[:, :, None]).reshape(-1, 18)
        B[:, 19] = Gb[:, 0] * vabs[0] + Gb[:, 1] * vabs[1] + Gb[:, 2] * vabs[2]
    return B


# --------------------------------------------------------------------------------------------------------------------
# records: [cost, gradC (18N, Eigen column-major d * 6N + 6i + q), gradT (N)]
# --------------------------------------------------------------------------------------------------------------------
def _acc_index(N):
    """Accumulator layout of outer_body / finalize_body: e = piece * 18 + 6d + q (gdC), 18N + piece (gdT), 19N (cost).
    Returns, for every accumulator entry < 18N, its position in the record (1 + d * 6N + 6i + q)."""
    e = np.arange(18 * N)
    piece, within = e // 18, e % 18
    d, q = within // 6, within % 6
    return 1 + d * 6 * N + 6 * piece + q


def _point_acc(terms: Terms):
    """[P, 20] per-point values in the interior-slot layout (cost, 18 gdC [d][q], gdT) and [P, 20] accumulator entries."""
    P, N = terms.piece.shape[0], terms.N
    vals = np.zeros((P, 20))
    vals[:, 0] = terms.pena
    vals[:, 1:19] = terms.gc.reshape(P, 18)
    vals[:, 19] = terms.gdT
    ent = np.zeros((P, 20), dtype=np.int64)
    ent[:, 0] = 19 * N
    ent[:, 1:19] = terms.piece[:, None] * 18 + np.arange(18)[None, :]
    ent[:, 19] = 18 * N + terms.piece
    return vals, ent


def _tot_to_record(tot, N):
    """finalize_body's last CTA: the record from the accumulator totals; gradT(j) = sum_{i = j+1}^{N-1} tot_gdT[i] from 0.0."""
    out = np.zeros(1 + 19 * N)
    out[0] = tot[19 * N]
    out[_acc_index(N)] = tot[: 18 * N]
    gT = tot[18 * N: 19 * N]
    for j in range(N):
        s = 0.0
        for i in range(j + 1, N):
            s = s + gT[i]
        out[1 + 18 * N + j] = s
    return out


def _entry_fsum(terms: Terms, V):
    """Per record entry, math.fsum of the per-point values V [P, 20] (cost, 18 gdC [d][q], gdT) over the active points that
    feed it: cost every point, gradC (i, d, q) the points of piece i, gradT (j) the points of pieces > j."""
    N = terms.N
    out = np.zeros(1 + 19 * N)
    a = terms.active
    out[0] = math.fsum(V[a, 0])
    pos = _acc_index(N).reshape(N, 18)
    for i in range(N):
        Vi = V[a & (terms.piece == i)]
        for w in range(18):
            out[pos[i, w]] = math.fsum(Vi[:, 1 + w])
    for j in range(N):
        out[1 + 18 * N + j] = math.fsum(V[a & (terms.piece > j), 19])
    return out


def exact_record(terms: Terms):
    """(record, abs_sum): every entry the exactly rounded sum of its terms (math.fsum) and sum |terms| per entry."""
    vals, _ = _point_acc(terms)
    return _entry_fsum(terms, vals), _entry_fsum(terms, np.abs(vals))


def bound_sum(terms: Terms):
    """sum of the terms' magnitude bounds B per entry (the FMA build's allowance, kappa * u * bound_sum)."""
    return _entry_fsum(terms, terms.B)


def _seq_sum(M, axis=-1):
    """Sum along `axis` strictly left to right, from +0.0."""
    M = np.moveaxis(np.asarray(M, dtype=np.float64), axis, -1)
    s = np.zeros(M.shape[:-1])
    for k in range(M.shape[-1]):
        s = s + M[..., k]
    return s


def _warp_tree(V):
    """warp_sum_fixed over the last axis (32 lanes): shuffle-down by 16, 8, 4, 2, 1, read at lane 0."""
    v = np.array(V, dtype=np.float64, copy=True)
    off = 16
    while off:
        v[..., :off] = v[..., :off] + v[..., off: 2 * off]
        off >>= 1
    return v[..., 0]


def _lane_strided(M):
    """finalize_body's loop `for (k = lane; k < n; k += 32) s += M[k]` then the shuffle tree, for every row of M [rows, n]."""
    rows, n = M.shape
    n32 = 32 * max(1, -(-n // 32))
    Z = np.zeros((rows, n32))
    Z[:, :n] = M
    return _warp_tree(_seq_sum(Z.reshape(rows, n32 // 32, 32), axis=1))


def is_batched(P, grid):
    return P >= BATCHED_MIN * grid * WARPS_PER_CTA


def warp_schedule(P, grid, batched):
    """[W, L] point indices (-1: none) in the order each warp of outer_body walks them."""
    W = grid * WARPS_PER_CTA
    if P == 0:
        return np.full((W, 0), -1, dtype=np.int64)
    if not batched:  # warp w: points w, w + W, ... (batches of 32 lanes, lane order = point order)
        L = -(-P // W)
        idx = np.arange(W)[:, None] + W * np.arange(L)[None, :]
        return np.where(idx < P, idx, -1)
    nB = W * (-(-P // (32 * W)))
    per_warp = nB // W
    bi = np.arange(W)[:, None] + W * np.arange(per_warp)[None, :]  # [W, per_warp] batches
    first, end = (bi * P) // nB, ((bi + 1) * P) // nB
    width = int((end - first).max())
    assert width <= 32
    lane = np.arange(width)
    idx = first[:, :, None] + lane[None, None, :]
    idx = np.where(idx < end[:, :, None], idx, -1)
    return idx.reshape(W, per_warp * width)


def ordered_record(terms: Terms, inside, grid, batched=None):
    """The record the kernels produce, restated in their order.  inside [P] bool: the points of the interior branch (their
    terms go through gsip_body's slots, the others through outer_body's warp accumulators).  batched: None = the runtime's
    rule.  Returns (record with n_inside appended, info) where info carries what gamma_bound needs."""
    N = terms.N
    P = terms.piece.shape[0]
    inside = np.asarray(inside, dtype=bool).reshape(P)
    if batched is None:
        batched = is_batched(P, grid)
    nacc = 19 * N + 1
    W = grid * WARPS_PER_CTA
    vals, ent = _point_acc(terms)
    # outer_body: each warp adds its active, non-interior points in order, one accumulator chain per entry
    sched = warp_schedule(P, grid, batched)
    acc = np.zeros((W, nacc))
    use = np.zeros(P, dtype=bool) if P == 0 else (terms.active & ~inside)
    chain = np.zeros(W, dtype=np.int64)
    rows = np.arange(W)
    for l in range(sched.shape[1]):
        k = sched[:, l]
        ok = k >= 0
        ok[ok] = use[k[ok]]
        r, kk = rows[ok], k[ok]
        e = ent[kk]
        acc[r[:, None], e] = acc[r[:, None], e] + vals[kk]
        chain[r] += 1
    # CTA partial: the 8 warps in order
    partials = _seq_sum(acc.reshape(grid, WARPS_PER_CTA, nacc), axis=1)  # [grid, nacc]
    s = _lane_strided(partials.T)  # [nacc]
    # interior slots, ascending point order; gradC / gradT entries take the slots of their own piece only
    slots = np.flatnonzero(inside)
    n_in = slots.size
    M = np.zeros((nacc, n_in))
    if n_in:
        sv = np.where(terms.active[slots][:, None], vals[slots], 0.0)
        pc = terms.piece[slots]
        pe = np.arange(18 * N) // 18
        M[: 18 * N] = np.where(pc[None, :] == pe[:, None], sv[:, 1 + np.arange(18 * N) % 18].T, 0.0)
        M[18 * N: 19 * N] = np.where(pc[None, :] == np.arange(N)[:, None], sv[:, 19][None, :], 0.0)
        M[19 * N] = sv[:, 0]
    s2 = _lane_strided(M)
    tot = s + s2
    out = np.r_[_tot_to_record(tot, N), float(n_in)]
    info = dict(grid=grid, batched=bool(batched), n_in=n_in, max_chain=int(chain.max()) if W else 0)
    return out, info


def chain_lengths(info, N):
    """h per record entry: the longest addition chain any term passes through.  Outer terms: the warp chain, 8 warps, the
    lane's ceil(grid / 32) partials, the 5-level tree; interior terms: ceil(n_in / 32) slots and the tree; then s + s2.
    gradT adds the suffix of up to N - 1 piece totals."""
    outer = info["max_chain"] + WARPS_PER_CTA + -(-info["grid"] // 32) + 5
    inner = -(-info["n_in"] // 32) + 5
    h = np.full(1 + 19 * N, max(outer, inner) + 1, dtype=np.int64)
    h[1 + 18 * N:] += N - 1
    return h


def gamma(h):
    h = np.asarray(h, dtype=np.float64)
    return h * U / (1.0 - h * U)


def gamma_bound(info, abs_sum, N):
    """gamma_h * sum |terms| per entry: |ordered - exact| is at most this for the schedule described by info."""
    return gamma(chain_lengths(info, N)) * np.asarray(abs_sum)


def bits_equal(a, b):
    """Bitwise equality of two float64 arrays (NaN payloads and signed zeros included)."""
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(np.array_equal(a.view(np.int64), b.view(np.int64)))


def oracle_order_record(terms: Terms):
    """The oracle's addSafetyPenaltyTrueSDF with one thread: every point in order, cost += pena,
    gradC[d * 6N + 6i + q] += beta_q G_d, gradT[j] += gdT for j < piece.  (Its inactive points add zeros: no change.)"""
    N = terms.N
    P = terms.piece.shape[0]
    out = np.zeros(1 + 19 * N)
    out[0] = _seq_sum(terms.pena[None, :])[0]
    vals = terms.gc.reshape(P, 18)
    pos = _acc_index(N)
    M = np.zeros((18 * N, P))
    e = terms.piece[:, None] * 18 + np.arange(18)[None, :]
    M[e.ravel(), np.repeat(np.arange(P), 18)] = vals.ravel()
    out[pos] = _seq_sum(M)
    MT = np.where(terms.piece[None, :] > np.arange(N)[:, None], terms.gdT[None, :], 0.0)
    out[1 + 18 * N:] = _seq_sum(MT)
    return out


def split_record(out, N):
    """(cost, gradC [18N], gradT [N]) of a record."""
    return out[0], out[1: 1 + 18 * N], out[1 + 18 * N: 1 + 19 * N]
