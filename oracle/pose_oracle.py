"""oracle/pose_oracle.py — TEST INFRASTRUCTURE ONLY (never imported by the product; tests/ compare the device kernels with it).

Python restatement of the pose-sampled obstacle penalty (svsdf_set_pose_penalty): the reference's grad_cost_p
(src/planner_algorithm/include/planner_algorithm/back_end_optimizer.hpp:956-1028) at the samples of addTimeIntPenalty (:411-533), on
k3_points.GridMap3D and the oracle's shape functors (oracle_py.shape_sdf / shape_grad1, the reference's getonlySDF / getonlyGrad1 bit for
bit), and the chain rule host::pose_penalty (csrc/host/minco.hpp) applies to the sample records.

Every expression is written in the grouping the kernel (csrc/svsdf_pose.cu, strict build) evaluates it in, with one IEEE rounding per
operation (Python floats and numpy element-wise operations do not contract a * b + c), so the strict kernel's records equal these bit for
bit.  The map's upper boundary is boundary_min + size * res (the device holds the map as kernel bytes, without the cloud's maximum), as
the query-point extraction takes it.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import oracle_py


def smoothed_l1(x: float, mu: float = 0.01):
    """smoothedL1 (back_end_optimizer.hpp:316-340): (active, f, df)."""
    if x < 0.0:
        return False, 0.0, 0.0
    if x > mu:
        return True, x - 0.5 * mu, 1.0
    xdmu = x / mu
    sqrxdmu = xdmu * xdmu
    mumxd2 = mu - 0.5 * x
    return True, mumxd2 * sqrxdmu * xdmu, sqrxdmu * ((-0.5) * xdmu + 3.0 * mumxd2 / mu)


def index_box(gm, centre, half):
    """map_index_box (svsdf_types.h): the clamped inclusive index box [(first, last)] * 3 around centre."""
    lo = gm.boundary_min
    size = gm.size
    out = []
    for a in range(3):
        hi = lo[a] + float(size[a]) * gm.res
        pair = []
        for side in (0, 1):
            v = centre[a] + (half[a] if side else -half[a])
            v = lo[a] if v < lo[a] else v
            v = hi if v > hi else v
            i = int(math.floor((v - lo[a]) / gm.res))
            i = 0 if i < 0 else i
            i = size[a] - 1 if i >= size[a] else i
            pair.append(i)
        out.append(tuple(pair))
    return out


def sample_pose(T, coeffs_colmajor, i, j, R):
    """addTimeIntPenalty's sample j of piece i: (s1, step, pos = c_i^T beta0(s1)) with the kernel's sums."""
    T = np.asarray(T, dtype=np.float64)
    c = np.asarray(coeffs_colmajor, dtype=np.float64).reshape(-1)
    N = T.shape[0]
    step = float(T[i]) * (1.0 / R)
    s1 = j * step
    s2 = s1 * s1
    s3 = s2 * s1
    s4 = s2 * s2
    s5 = s4 * s1
    b0 = (1.0, s1, s2, s3, s4, s5)
    pos = []
    for d in range(3):
        a = 0.0
        for q in range(6):
            a += float(c[d * 6 * N + 6 * i + q]) * b0[q]
        pos.append(a)
    return s1, step, pos


def grad_cost_p(gm, shape, pos, half, safety_hor, poly_params=(0.0, 0.0, 0.0), polygon=None, with_cells=False):
    """One sample's record (costp, gradp_x, gradp_y, grad_yaw): grad_cost_p with rotate's unset entries 0, the pinned sincos, the voxels
    in getPointsInAABB's order (i, j, k ascending, k innermost) and the box filter |p_rel_a| > half_a (equality kept).  with_cells: also
    the (i, j, k) of the cells that passed the filter and of those that were active."""
    sy_a, cy_a = oracle_py.sincos(np.array([pos[2]]))
    sy, cy = float(sy_a[0]), float(cy_a[0])
    box = index_box(gm, pos, half)
    cells = [(i, j, k) for i in range(box[0][0], box[0][1] + 1) for j in range(box[1][0], box[1][1] + 1)
             for k in range(box[2][0], box[2][1] + 1) if gm.occ[i, j, k]]
    lo = gm.boundary_min
    kept = []
    for (i, j, k) in cells:
        cx = (i + 0.5) * gm.res + lo[0]
        cyy = (j + 0.5) * gm.res + lo[1]
        cz = (k + 0.5) * gm.res + lo[2]
        d0, d1, d2 = cx - pos[0], cyy - pos[1], cz - pos[2]
        rx = cy * d0 + sy * d1
        ry = (-sy) * d0 + cy * d1
        if abs(rx) > half[0] or abs(ry) > half[1] or abs(d2) > half[2]:
            continue
        kept.append((i, j, k, d0, d1, rx, ry))
    costp = gpx = gpy = gyaw = 0.0
    active = []
    if kept:
        rel = np.array([[e[5], e[6], 0.0] for e in kept])
        if shape == "Circle":  # getSDFwithGrad1's value leaves poly_params out (Shape.hpp:497-503)
            sdf = oracle_py.shape_sdf(shape, rel, (0.0, 0.0, 0.0), polygon)
        else:
            sdf = oracle_py.shape_sdf(shape, rel, poly_params, polygon)
        g = oracle_py.shape_grad1(shape, rel, poly_params, polygon)
        for n, (i, j, k, d0, d1, rx, ry) in enumerate(kept):
            on, f, L1 = smoothed_l1(safety_hor - float(sdf[n]), 0.01)
            if not (on and f > 0):
                continue
            gx, gy = float(g[n, 0]), float(g[n, 1])
            rg0 = -(cy * gx + (-sy) * gy)
            rg1 = -(sy * gx + cy * gy)
            w0 = (-sy) * d0 + cy * d1
            w1 = (-cy) * d0 + (-sy) * d1
            costp += f
            gpx += (-L1) * rg0
            gpy += (-L1) * rg1
            gyaw += ((-L1) * gx) * w0 + ((-L1) * gy) * w1
            active.append((i, j, k))
    rec = (costp, gpx, gpy, gyaw)
    if with_cells:
        return rec, [(e[0], e[1], e[2]) for e in kept], active
    return rec


def records(gm, shape, T, coeffs_colmajor, R, half, safety_hor, poly_params=(0.0, 0.0, 0.0), polygon=None):
    """Every sample's record, [N (R + 1), 4], piece-major (svsdf_pose_penalty_eval's samples_out)."""
    N = len(T)
    out = np.zeros((N * (R + 1), 4))
    for i in range(N):
        for j in range(R + 1):
            _, _, pos = sample_pose(T, coeffs_colmajor, i, j, R)
            out[i * (R + 1) + j] = grad_cost_p(gm, shape, pos, half, safety_hor, poly_params, polygon)
    return out


def accumulate(weight, R, T, coeffs_colmajor, rec):
    """host::pose_penalty: (cost, gradT [N], gradC [18N column-major]) from the sample records, in its summation order."""
    T = np.asarray(T, dtype=np.float64)
    b = np.asarray(coeffs_colmajor, dtype=np.float64).reshape(-1)
    rec = np.asarray(rec, dtype=np.float64).reshape(-1, 4)
    N = T.shape[0]
    n = 6 * N
    gC = [0.0] * (18 * N)
    gT = [0.0] * N
    partial = [0.0] * N
    frac = 1.0 / R
    for i in range(N):
        step = float(T[i]) * frac
        part = 0.0
        for j in range(R + 1):
            r = rec[i * (R + 1) + j]
            if not (r[0] > 0.0):
                continue
            gP = (weight * float(r[1]), weight * float(r[2]), weight * float(r[3]))
            pena = weight * float(r[0])
            s1 = j * step
            s2 = s1 * s1
            s3 = s2 * s1
            s4 = s2 * s2
            s5 = s4 * s1
            node = 0.5 if (j == 0 or j == R) else 1.0
            alpha = j * frac
            dot = 0.0
            for d in range(3):
                c = [float(v) for v in b[d * n + 6 * i: d * n + 6 * i + 6]]
                vel = c[1] + 2.0 * s1 * c[2] + 3.0 * s2 * c[3] + 4.0 * s3 * c[4] + 5.0 * s4 * c[5]
                dot = gP[0] * vel if d == 0 else dot + gP[d] * vel
                o = d * n + 6 * i
                for k, bk in enumerate((1.0, s1, s2, s3, s4, s5)):
                    gC[o + k] += bk * gP[d] * node * step
            gT[i] += dot * alpha * node * step + node * frac * pena
            part += node * step * pena
        partial[i] = part
    cost = 0.0
    for i in range(N):
        cost += partial[i]
    return cost, np.array(gT), np.array(gC)


def pose_penalty(gm, shape, T, coeffs_colmajor, weight, R, half, safety_hor, poly_params=(0.0, 0.0, 0.0), polygon=None):
    """(cost, gradT, gradC, records) of one trajectory: records() then accumulate()."""
    rec = records(gm, shape, T, coeffs_colmajor, R, half, safety_hor, poly_params, polygon)
    cost, gT, gC = accumulate(weight, R, T, coeffs_colmajor, rec)
    return cost, gT, gC, rec
