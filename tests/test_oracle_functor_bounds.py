"""CPU checks of the arguments behind two exactness shortcuts of the shape functors (SURVEY.md §8a rows A3 and A9).

1. Mesh far-field bound.  choiceTInit's layer 1 skips a lattice sample when |q| >= prune_rmin and
   sdf >= (|q| - rout) / prune_scale already exceeds the best value found.  For the mesh functor svsdf_create derives
   prune_rmin = rho0, rout ~ Rv and prune_scale = 1 / (1 - 2 omega) from the root of the winding-number hierarchy
   (csrc/svsdf_runtime_context.cpp, upload_mesh's "Far-field bound" block): omega is a term-by-term bound of the root children's order-2
   expansions beyond rho0.  It is restated here in numpy from api.mesh_fwn_host's children and rows and checked against the
   oracle's float winding number (bitwise the reference's): |w(q)| <= omega on dense rings of z = 0 points at
   |q| = rho0 (1 + 1e-6), 1.5 rho0 and 10 rho0, and sdf(q) >= (1 - 2 omega)(|q| - Rv) there.  Where omega >= 0.45 or is not
   finite the library leaves the pruning off (rout stays 1e300, build_shape); the restatement must say so for that mesh.

2. Polygon crossing test.  polygon_scan (csrc/svsdf_shapes.cuh) decides the reference's |ths - the| >= pi by sign tests and
   calls atan2 only when an offset lies exactly on the horizontal through q or the two offsets are within a relative 1e-9 of
   (anti)parallel.  polygon_cases() builds point sets aimed at that switch (tests/test_gpu_functor_edges.py runs them through
   the device functor bit for bit); the tests here prove that each set reaches both sides of it, and that wherever the sign
   tests decide they agree with the angles.

The mesh and polygon builders below are shared with tests/test_gpu_functor_edges.py."""
import json
import os
import sys

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, scenes

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
sys.path.insert(0, GOLD)
import make_live_golden as mkl  # noqa: E402  (the builder-branch meshes of the winding-number comparison)

EMPTY, INTERNAL = 0xFFFFFFFF, 0x80000000
PRUNE_OMEGA_MAX = 0.45  # svsdf_create enables the pruning only below this


# ---------------------------------------------------------------------------------------------------------------------
# meshes
# ---------------------------------------------------------------------------------------------------------------------
def golden_mesh(name):
    g = np.load(os.path.join(GOLD, "fwn_ref_sdarc.npz" if name == "sdArc" else "fwn_ref.npz"))
    return g[name + "_V"], g[name + "_F"]


def open_triangle():
    """One large triangle, tilted out of the z = 0 plane: an open mesh."""
    V = np.array([[-3.0, -2.0, -0.4], [4.0, -1.0, 0.3], [0.5, 3.5, 0.8]])
    return V, np.array([[0, 1, 2]], dtype=np.int32)


def open_box():
    """An axis-aligned box 4 x 2 x 1 with its +x side missing (10 outward faces): an open mesh with |w| up to 1/2 near it."""
    V = np.array([[x, y, z] for x in (-2.0, 2.0) for y in (-1.0, 1.0) for z in (-0.5, 0.5)])
    quads = [(0, 1, 3, 2), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]  # the +x quad (4, 6, 7, 5) is left out
    F = []
    for a, b, c, d in quads:
        F += [[a, b, c], [a, c, d]]
    return V, np.asarray(F, dtype=np.int32)


def bound_cases():
    """name -> (V, F, poly_params) of the far-field bound check.  poly_params carry translations only, so that the numpy
    restatement of svsdf_create's vertex transform is exact (R = I)."""
    star = golden_mesh("star")
    cases = {"star_obj": (*star, (0.0, 0.0, 0.0)), "sdHorseshoe_obj": (*golden_mesh("sdHorseshoe"), (0.0, 0.0, 0.0)),
             "sdArc_obj": (*golden_mesh("sdArc"), (0.0, 0.0, 0.0))}
    for m in mkl.FWN_MESHES:
        V, F, _ = mkl.fwn_mesh(m)
        cases["fwn_" + m] = (V, F, (0.0, 0.0, 0.0))
    cases["open_triangle"] = (*open_triangle(), (0.0, 0.0, 0.0))
    cases["open_box"] = (*open_box(), (0.0, 0.0, 0.0))
    cases["star_obj_off_origin"] = (*star, (5.0, -3.0, 0.0))
    cases["star_obj_x1e-3"] = (star[0] * 1e-3, star[1], (0.0, 0.0, 0.0))
    cases["star_obj_x1e3"] = (star[0] * 1e3, star[1], (0.0, 0.0, 0.0))
    return cases


def shape_frame_vertices(V, pp):
    """svsdf_create's vertex transform ((v0 R[j][0] + v1 R[j][1]) + v2 R[j][2]) + tr[j] for R = I: v + (tx, ty, 0)."""
    assert pp[2] == 0.0
    Vt = np.asarray(V, dtype=np.float64).copy()
    Vt[:, 0] = Vt[:, 0] + pp[0]
    Vt[:, 1] = Vt[:, 1] + pp[1]
    return Vt


def far_field_bound(V, F, pp=(0.0, 0.0, 0.0)):
    """(Rv, rho0, omega, finite) exactly as svsdf_create computes them, from the library's own hierarchy."""
    Vt = shape_frame_vertices(V, pp)
    ch, data, _ = api.mesh_fwn_host(Vt, F)
    row = data[0].astype(np.float64)  # [23][4]: root record, lane i = child i
    Rv = float(np.max(np.sqrt((Vt[:, 0] * Vt[:, 0] + Vt[:, 1] * Vt[:, 1]) + Vt[:, 2] * Vt[:, 2])))
    nchild = 0
    while nchild < 4 and ch[0, nchild] != EMPTY:
        nchild += 1
    Pn = np.sqrt((row[1] * row[1] + row[2] * row[2]) + row[3] * row[3])
    rho0 = 0.0
    for i in range(nchild):
        rho0 = max(rho0, Pn[i] + 2.0 * np.sqrt(max(0.0, row[0, i])))
    rho0 = max(rho0, Rv) * (1.0 + 1e-4) + 1e-6
    a = np.abs(row)
    omega, finite = 0.0, bool(np.isfinite(rho0))
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        for i in range(nchild):
            if not finite:
                break
            m = 1.0 / (rho0 - Pn[i])
            A0 = a[4, i] + a[5, i] + a[6, i]
            A1 = abs(row[7, i] + row[8, i] + row[9, i]) + 3.0 * (a[7, i] + a[8, i] + a[9, i] + a[10, i] + a[11, i] + a[12, i])
            t0 = abs(row[20, i] + row[21, i]) + abs(row[22, i] + row[17, i]) + abs(row[18, i] + row[19, i])
            t1 = a[17, i] + a[18, i] + a[19, i] + a[20, i] + a[21, i] + a[22, i]
            A2 = 1.5 * (3.0 * (a[13, i] + a[14, i] + a[15, i]) + t0) + 7.5 * (a[13, i] + a[14, i] + a[15, i] + a[16, i] + t1)
            omega += A0 * m * m + A1 * m * m * m + A2 * m * m * m * m
            finite = finite and bool(np.isfinite(omega))
    omega = omega / (4.0 * np.pi) * 1.02 + 1e-6
    return Rv, rho0, omega, finite


def ring(r, n=20_000, phase=0.0):
    th = phase + 2.0 * np.pi * np.arange(n) / n
    return np.c_[r * np.cos(th), r * np.sin(th), np.zeros(n)]


# ---------------------------------------------------------------------------------------------------------------------
# polygons
# ---------------------------------------------------------------------------------------------------------------------
def star_obj_outline():
    """Config 4's polygon: the outline of shapes/star.obj (40 vertices), ordered by angle as tests/test_gpu_gsip.py builds it."""
    xy = np.array(json.load(open(os.path.join(GOLD, "obj_outlines.json")))["star"]["outline_xy"])
    return xy[np.argsort(np.arctan2(xy[:, 1], xy[:, 0]))]


def polygons():
    """name -> vertices [n, 2] of the Polygon functor cases."""
    star = star_obj_outline()
    return {
        "star_obj_outline": star,
        "star_obj_outline_cw": star[::-1].copy(),
        "collinear_three": np.array([[-2.0, -1.0], [0.0, -1.0], [2.0, -1.0], [2.0, 1.5], [-0.5, 2.0], [-2.0, 1.0]]),
        "repeated_vertex": np.array([[3.0, -1.0], [3.0, 1.0], [3.0, 1.0], [0.0, 2.5], [-3.0, 1.0], [-3.0, -1.0]]),
        "bow_tie": np.array([[-2.0, -1.0], [2.0, 1.0], [2.0, -1.0], [-2.0, 1.0]]),
        "near_1e6": np.array([[3.0, -1.0], [3.0, 1.0], [0.0, 2.5], [-3.0, 1.0], [-3.0, -1.0]]) * 0.7 + np.array([1.0e6, -1.0e6 + 0.25]),
    }


def _ulp_steps(v, ks=(1, 2, 4)):
    out = [v]
    for k in ks:
        up = dn = v
        for _ in range(k):
            up, dn = np.nextafter(up, np.inf), np.nextafter(dn, -np.inf)
        out += [up, dn]
    return out


def polygon_cases(P):
    """Points [m, 3] (z = 0) aimed at polygon_scan's switch between the sign tests and atan2 for polygon P."""
    P = np.asarray(P, dtype=np.float64)
    n = len(P)
    c = P.mean(axis=0)
    scale = float(np.max(np.abs(P - c)))
    pts = []
    # q.y equal to a vertex's y and its 1, 2 and 4 ulp neighbours, q.x left of, right of, near and far from the polygon
    dx = np.array([-3.1, -1.3, -0.21, 0.0, 0.37, 1.1, 2.9]) * scale
    for v in P:
        for y in _ulp_steps(v[1]):
            for x in np.r_[v[0] + dx, c[0] + dx]:
                pts.append((x, y))
    # q at every vertex
    pts += [tuple(v) for v in P]
    for i in range(n):
        s, e = P[i], P[(i + 1) % n]
        d = e - s
        L = float(np.hypot(d[0], d[1]))
        if L == 0.0:
            continue
        nrm = np.array([-d[1], d[0]]) / L
        for lam in (-2.5, -1.0, -0.3, -1e-3, 0.1, 0.5, 0.77, 1.0 + 1e-3, 1.3, 3.0):
            q = s + lam * d  # on the supporting line, inside and outside the segment (double rounding)
            pts.append(tuple(q))
            # a and b = s - q, e - q at a relative rho of (anti)parallel: |cross(a, b)| = rho |lam (1 - lam)| |d|^2
            for rho in (1e-10, 1e-9, 3e-9, 1e-8):
                for sg in (1.0, -1.0):
                    pts.append(tuple(q + sg * rho * abs(lam * (1.0 - lam)) * L * nrm))
    # the outline's symmetry axes (for the star: the lines through the origin and each tip / notch; for every polygon the
    # lines through its centre and each vertex and edge midpoint, and the two coordinate axes through the centre)
    dirs = [P[i] - c for i in range(n)] + [(P[i] + P[(i + 1) % n]) / 2 - c for i in range(n)] + [np.array([1.0, 0.0]), np.array([0.0, 1.0])]
    ts = np.array([-1.7, -1.0, -0.6, 0.0, 0.45, 0.99, 1.0, 1.01, 1.6, 4.0])
    for u in dirs:
        nu = float(np.hypot(u[0], u[1]))
        if nu == 0.0:
            continue
        u = u / nu * scale
        for t in ts:
            pts.append(tuple(c + t * u))
    Q = np.array(pts, dtype=np.float64)
    return np.c_[Q, np.zeros(len(Q))]


def scan_branches(P, Q):
    """polygon_scan's branch condition restated: per (point, edge) the offsets a = s - q, b = e - q, cr = cross(a, b), the
    threshold 1e-9 (|a|_1 |b|_1) and whether the atan2 branch is taken."""
    P = np.asarray(P, dtype=np.float64)
    S, E = P, np.roll(P, -1, axis=0)
    qx, qy = Q[:, :1], Q[:, 1:2]
    ax, ay, bx, by = S[:, 0] - qx, S[:, 1] - qy, E[:, 0] - qx, E[:, 1] - qy
    cr = ax * by - ay * bx
    thr = 1e-9 * ((np.abs(ax) + np.abs(ay)) * (np.abs(bx) + np.abs(by)))
    use_atan2 = ~((ay != 0.0) & (by != 0.0) & (np.abs(cr) > thr))
    return ax, ay, bx, by, cr, thr, use_atan2


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(bound_cases()))
def test_mesh_far_field_bound_holds(oracle_mod, name):
    """|w| <= omega beyond rho0 and sdf >= (1 - 2 omega)(|q| - Rv) on 3 x 20 000 z = 0 points per mesh."""
    V, F, pp = bound_cases()[name]
    Rv, rho0, omega, finite = far_field_bound(V, F, pp)
    if not (finite and omega < PRUNE_OMEGA_MAX):
        # the library then keeps rout = 1e300 (build_shape): no layer-1 sample of this mesh is ever pruned
        print(f"{name}: omega = {omega:.4g} (finite {finite}): pruning off")
        assert not finite or omega >= PRUNE_OMEGA_MAX
        return
    worst, slack_sdf = 0.0, np.inf
    for k, r in enumerate((rho0 * (1.0 + 1e-6), 1.5 * rho0, 10.0 * rho0)):
        Q = ring(r, phase=0.37 * k)
        w = oracle_mod.mesh_eval((V, F), Q, "winding", poly_params=pp)
        assert np.all(np.isfinite(w))
        worst = max(worst, float(np.abs(w).max()))
        sdf = oracle_mod.mesh_eval((V, F), Q, "sdf", poly_params=pp)
        lower = (1.0 - 2.0 * omega) * (np.hypot(Q[:, 0], Q[:, 1]) - Rv)
        assert np.all(sdf >= lower), (name, r, float((lower - sdf).max()))
        slack_sdf = min(slack_sdf, float((sdf - lower).min()))
    s = omega - worst
    print(f"{name}: Rv {Rv:.6g} rho0 {rho0:.6g} omega {omega:.4g} max|w| {worst:.4g} slack {s:.4g} ({s / omega:.1%} of omega); "
          f"sdf slack {slack_sdf:.4g}")
    assert worst <= omega, (name, worst, omega)


def test_far_field_bound_restatement_sees_both_outcomes():
    """The case list is not vacuous: the meshes the planner runs get a finite omega < 0.45, so their pruning is on and the
    bound above is what keeps it exact.  (Every mesh of the list does, the open ones included.)"""
    res = {n: far_field_bound(*c) for n, c in bound_cases().items()}
    on = [n for n, (_, _, om, fin) in res.items() if fin and om < PRUNE_OMEGA_MAX]
    assert {"star_obj", "sdHorseshoe_obj", "sdArc_obj", "star_obj_x1e3", "star_obj_off_origin"} <= set(on), res
    # the bound scales: the same mesh 1e3 or 1e-3 times larger has nearly the same omega (the absolute 1e-6 pads of rho0
    # and omega are 1.6e-4 and 6e-6 of them at 1e-3 scale)
    om = res["star_obj"][2]
    for n in ("star_obj_x1e3", "star_obj_x1e-3"):
        assert abs(res[n][2] - om) <= 1e-3 * om, (n, res[n][2], om)


@pytest.mark.parametrize("name", list(polygons()))
def test_polygon_cases_reach_both_branches(name):
    """Each polygon's point set sends >= 100 points down the atan2 branch and >= 100 down the sign branch with |cr| within a
    factor of 10 of the threshold."""
    P = polygons()[name]
    Q = polygon_cases(P)
    _, _, _, _, cr, thr, use_atan2 = scan_branches(P, Q)
    n_atan2 = int(use_atan2.any(axis=1).sum())
    near = ~use_atan2 & (np.abs(cr) <= 10.0 * thr)
    n_near = int(near.any(axis=1).sum())
    print(f"{name}: {len(Q)} points, {n_atan2} take the atan2 branch on some edge, {n_near} the sign branch within 10x of "
          f"the threshold")
    assert n_atan2 >= 100 and n_near >= 100, (n_atan2, n_near)


@pytest.mark.parametrize("name", list(polygons()))
def test_polygon_sign_tests_agree_with_the_angles(name):
    """Wherever polygon_scan uses the sign tests, they give the reference's |ths - the| >= pi decision: the angles are taken
    in double by numpy (any faithful atan2 decides the same way there, the margin being >= 1e-9 rad), on the adversarial
    set and on 20 000 random points around the polygon."""
    P = polygons()[name]
    c, scale = P.mean(axis=0), float(np.max(np.abs(P - P.mean(axis=0))))
    rng = np.random.default_rng(71)
    R = np.c_[c + rng.uniform(-2.0, 2.0, size=(20_000, 2)) * scale, np.zeros(20_000)]
    Q = np.r_[polygon_cases(P), R]
    ax, ay, bx, by, cr, thr, use_atan2 = scan_branches(P, Q)
    sign = ((ay > 0.0) != (by > 0.0)) & np.where(ay > 0.0, cr < 0.0, cr > 0.0)
    ths, the = np.arctan2(ay, ax), np.arctan2(by, bx)
    ths = np.where(ths < 0.0, ths + 2 * np.pi, ths)
    the = np.where(the < 0.0, the + 2 * np.pi, the)
    ang = ~(np.abs(ths - the) < np.pi)
    sel = ~use_atan2
    assert np.array_equal(sign[sel], ang[sel]), int((sign[sel] != ang[sel]).sum())
