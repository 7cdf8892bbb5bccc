"""CPU: the swept-volume contour checker (oracle/swept_oracle.hpp) against the svsdf_swept_contour contract — every marching-squares
case written out by hand, the inside convention, closed and oriented loops, the fill against the outline, watertight prisms, and grids
of different boxes that line up."""
import math

import numpy as np
import pytest

from implicit_svsdf_planner_b200.api import SweptContour, write_prism_obj
from oracle import swept_py

# unit cell, iso 0, inside corners -1 and outside corners +1: every crossing at the edge midpoint
C0, C1, C2, C3 = (0.0, 0.0), (1.0, 0.0), (1.0, 1.0), (0.0, 1.0)
E0, E1, E2, E3 = (0.5, 0.0), (1.0, 0.5), (0.5, 1.0), (0.0, 0.5)
# case (bit k = corner ck inside) -> inside polygons, counter-clockwise from the walk's first item (c0, e0, c1, e1, c2, e2, c3, e3)
HAND = {
    0: [],
    1: [[C0, E0, E3]],
    2: [[E0, C1, E1]],
    3: [[C0, C1, E1, E3]],
    4: [[E1, C2, E2]],
    5: [[C0, E0, E1, C2, E2, E3]],          # connected saddle (m <= iso)
    6: [[E0, C1, C2, E2]],
    7: [[C0, C1, C2, E2, E3]],
    8: [[E2, C3, E3]],
    9: [[C0, E0, E2, C3]],
    10: [[E0, C1, E1, E2, C3, E3]],         # connected saddle
    11: [[C0, C1, E1, E2, C3]],
    12: [[E1, C2, C3, E3]],
    13: [[C0, E0, E1, C2, C3]],
    14: [[E0, C1, C2, C3, E3]],
    15: [[C0, C1, C2, C3]],
}
EDGES = {E0, E1, E2, E3}


def field2x2(case, vin=-1.0, vout=1.0):
    """[row b][column a]: corner c0 = (0, 0), c1 = (1, 0), c3 = (0, 1), c2 = (1, 1)."""
    v = [vin if case >> k & 1 else vout for k in range(4)]
    return np.array([[v[0], v[1]], [v[3], v[2]]])


def expected(polys):
    segs, tris = [], []
    for p in polys:
        n = len(p)
        segs += [(p[k], p[(k + 1) % n]) for k in range(n) if p[k] in EDGES and p[(k + 1) % n] in EDGES]
        tris += [(p[0], p[k], p[k + 1]) for k in range(1, n - 1)]
    return segs, tris


def as_xy(r):
    V = [tuple(v) for v in r.vertices.tolist()]
    return V, [(V[a], V[b]) for a, b in r.segments.tolist()], [tuple(V[i] for i in t) for t in r.triangles.tolist()]


def vertex_order(case):
    """Horizontal crossings (row-major), vertical crossings, inside corners (row-major)."""
    ins = [case >> k & 1 for k in range(4)]
    out = [E0] if ins[0] != ins[1] else []
    out += [E2] if ins[3] != ins[2] else []
    out += [E3] if ins[0] != ins[3] else []
    out += [E1] if ins[1] != ins[2] else []
    out += [c for c, k in ((C0, 0), (C1, 1), (C3, 3), (C2, 2)) if ins[k]]
    return out


@pytest.mark.parametrize("case", range(16))
def test_every_case_by_hand(case):
    r = swept_py.swept_contour(field2x2(case), 0, 0, 1.0, 0.0)
    V, S, F = as_xy(r)
    assert V == vertex_order(case)
    segs, tris = expected(HAND[case])
    assert S == segs and F == tris
    assert r.clipped == int(case != 0)  # every corner of a 2 x 2 grid is on the border


def test_separated_saddles_by_hand():
    # m = ((-0.5 + 1) + (1 - 0.5)) / 4 = 0.25 > 0: each inside corner keeps its own triangle, s = 0.5 / 1.5 from the inside corner
    t = 1.0 / 3.0
    r = swept_py.swept_contour(field2x2(5, -0.5, 1.0), 0, 0, 1.0, 0.0)
    V, S, F = as_xy(r)
    e0, e2, e3, e1 = (t, 0.0), (2.0 / 3.0, 1.0), (0.0, t), (1.0, 2.0 / 3.0)
    assert V == [e0, e2, e3, e1, C0, C2]
    assert S == [(e0, e3), (e2, e1)]
    assert F == [(C0, e0, e3), (e1, C2, e2)]
    r = swept_py.swept_contour(field2x2(10, -0.5, 1.0), 0, 0, 1.0, 0.0)
    V, S, F = as_xy(r)
    e0, e2, e3, e1 = (2.0 / 3.0, 0.0), (t, 1.0), (0.0, 2.0 / 3.0), (1.0, t)
    assert S == [(e1, e0), (e3, e2)]
    assert F == [(e0, C1, e1), (e2, C3, e3)]
    # m exactly iso connects: ((-1 + 1) + (1 - 1)) / 4 = 0 <= 0
    for case in (5, 10):
        r = swept_py.swept_contour(field2x2(case, -1.0, 1.0), 0, 0, 1.0, 0.0)
        assert len(r.triangles) == 4 and len(r.segments) == 2
    # and m below iso connects too (inside -1, outside 0.5)
    r = swept_py.swept_contour(field2x2(5, -1.0, 0.5), 0, 0, 1.0, 0.0)
    assert len(r.triangles) == 4


def test_value_equal_to_iso_is_inside():
    r = swept_py.swept_contour(np.array([[0.25, 1.0], [1.0, 1.0]]), 0, 0, 1.0, 0.25)
    V, S, F = as_xy(r)
    assert V == [(0.0, 0.0), (0.0, 0.0), (0.0, 0.0)]  # s = 0: both crossings sit on the inside corner
    assert len(F) == 1 and len(S) == 1


def lattice(i0, j0, nx, ny, h):
    x = np.arange(i0, i0 + nx, dtype=np.int64).astype(np.float64) * h
    y = np.arange(j0, j0 + ny, dtype=np.int64).astype(np.float64) * h
    return np.meshgrid(x, y)  # [ny, nx]


def disc(h, r=1.3, c=(0.05, -0.02), hole=None, pad=0.5):
    i0, j0 = math.floor((c[0] - r - pad) / h), math.floor((c[1] - r - pad) / h)
    n = int(math.ceil((2 * r + 2 * pad) / h)) + 2
    X, Y = lattice(i0, j0, n, n, h)
    f = np.hypot(X - c[0], Y - c[1]) - r
    if hole is not None:
        f = np.maximum(f, hole - np.hypot(X - c[0], Y - c[1]))
    return f, i0, j0


def contour(f, i0, j0, h, iso=0.0):
    o = swept_py.swept_contour(f, i0, j0, h, iso)
    return SweptContour(i0, j0, f.shape[1], f.shape[0], h, iso, o.vertices, o.segments, o.triangles, o.clipped, f.size)


def signed_area(V, loop):
    p = V[loop[:-1]]
    q = V[loop[1:]]
    return 0.5 * np.sum(p[:, 0] * q[:, 1] - q[:, 0] * p[:, 1])


def tri_area(r):
    a, b, c = (r.vertices[r.triangles[:, k]] for k in range(3))
    return 0.5 * ((b[:, 0] - a[:, 0]) * (c[:, 1] - a[:, 1]) - (c[:, 0] - a[:, 0]) * (b[:, 1] - a[:, 1]))


@pytest.mark.parametrize("hole", [None, 0.6])
def test_disc_and_annulus_loops_orientation_and_areas(hole):
    h = 0.05
    r = contour(*disc(h, hole=hole), h)
    assert r.clipped == 0
    loops = r.loops()
    assert len(loops) == (1 if hole is None else 2)
    assert all(l[0] == l[-1] for l in loops)  # closed
    areas = sorted(signed_area(r.vertices, l) for l in loops)
    assert areas[-1] > 0  # outer loop counter-clockwise
    if hole is not None:
        assert areas[0] < 0  # hole clockwise
    ta = tri_area(r)
    assert np.all(ta >= -1e-15)
    assert abs(r.area() - ta.sum()) <= 1e-12 * abs(r.area())
    exact = math.pi * (1.3 ** 2 - (0.6 ** 2 if hole else 0.0))
    assert abs(r.area() - exact) < 0.01 * exact


def test_area_error_is_second_order():
    errs = []
    for h in (0.1, 0.05, 0.025):
        r = contour(*disc(h), h)
        errs.append(abs(r.area() - math.pi * 1.3 ** 2))
    assert errs[1] < errs[0] / 2.5 and errs[2] < errs[1] / 2.5, errs


def boundary_edges(tris):
    count = {}
    for t in tris.tolist():
        for k in range(3):
            e = (t[k], t[(k + 1) % 3])
            count[e] = count.get(e, 0) + 1
    return {e for e in count if (e[1], e[0]) not in count}


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_fill_boundary_is_the_segment_set_and_the_prism_is_watertight(seed, tmp_path):
    rng = np.random.default_rng(seed)
    h = 0.1
    X, Y = lattice(-30, -30, 61, 61, h)
    f = np.full(X.shape, 1.0)
    for _ in range(6):  # blobs that touch, merge and leave holes and saddles
        c, rad = rng.uniform(-2, 2, 2), rng.uniform(0.3, 1.2)
        f = np.minimum(f, np.hypot(X - c[0], Y - c[1]) - rad)
    f = np.maximum(f, 0.25 - np.hypot(X - 0.3, Y + 0.2))
    f[0, :] = f[-1, :] = f[:, 0] = f[:, -1] = 1.0
    r = contour(f, -30, -30, h, 0.0)
    assert r.clipped == 0
    assert boundary_edges(r.triangles) == {tuple(s) for s in r.segments.tolist()}
    assert len({tuple(s) for s in r.segments.tolist()}) == len(r.segments)
    path = tmp_path / "prism.obj"
    write_prism_obj(str(path), r, 0.0, 0.5)
    faces = [tuple(int(w) - 1 for w in line.split()[1:]) for line in open(path) if line.startswith("f ")]
    edges = {}
    for t in faces:
        for k in range(3):
            e = (t[k], t[(k + 1) % 3])
            edges[e] = edges.get(e, 0) + 1
    # every directed edge once and its reverse once: each edge belongs to exactly two faces, consistently oriented
    assert all(v == 1 for v in edges.values()) and all((b, a) in edges for a, b in edges)


def test_sub_box_is_the_restriction_of_the_larger_box():
    h = 0.05
    f, i0, j0 = disc(h)
    big = swept_py.swept_contour(f, i0, j0, h, 0.0)
    a0, b0, na, nb = 7, 11, 30, 25  # a sub-box that cuts the disc
    sub = swept_py.swept_contour(f[b0:b0 + nb, a0:a0 + na], i0 + a0, j0 + b0, h, 0.0)
    assert sub.clipped == 1

    def tris_in(r, lo, hi):
        V = r.vertices
        out = []
        for t in r.triangles.tolist():
            p = V[t]
            c = p.mean(axis=0)
            if np.all(c > lo) and np.all(c < hi):
                out.append(tuple(map(tuple, p.tolist())))
        return out

    lo = np.array([(i0 + a0) * h, (j0 + b0) * h])
    hi = np.array([(i0 + a0 + na - 1) * h, (j0 + b0 + nb - 1) * h])
    assert tris_in(sub, lo, hi) == tris_in(big, lo, hi)
    assert len(tris_in(sub, lo, hi)) == len(sub.triangles) > 0
    # the lattice is the same whatever the box: fl(i h) with no origin add
    assert np.array_equal(sub.vertices[:0], big.vertices[:0])


def test_nan_corners_are_not_evaluated():
    f = field2x2(15)
    f[0, 0] = np.nan
    r = swept_py.swept_contour(f, 0, 0, 1.0, 0.0)
    assert len(r.triangles) == 0 and len(r.segments) == 0 and len(r.vertices) == 3  # the three inside corners only
