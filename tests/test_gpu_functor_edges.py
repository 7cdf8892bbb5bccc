"""GPU tests of the shape functors' exactness shortcuts at their edges (run with -m gpu on an H100).

Four places in the device functors replace the reference's arithmetic by a cheaper computation that is argued to give the
same bits; these tests feed them the inputs where the argument could fail:

* polygon_scan's crossing test decides |ths - the| >= pi by sign tests, calling atan2 only next to the switch: the point
  sets of tests/test_oracle_functor_bounds.py (exact horizontals, supporting lines, vertices, 1e-9 / 1e-10 of parallel,
  symmetry axes) on six polygons, through Context.shape_sdf and shape_grad1, bit for bit against the oracle (same pinned
  atan2).
* the mesh functor on every branch of the hierarchy builder: (1 - 2 w) sqrt(d2) with the oracle's float winding number w,
  which tests/golden/ref_live.npz ties to the reference's own code.
* closest_sqr_distance's pruned, nearest-first descent (float box lower bounds, bestf, the squared z gap, an explicit
  stack): the device distance must be the plain minimum over all faces.  Strict build: bitwise the oracle's brute force.
  Both builds: against the exact point-triangle distance (fractions.Fraction on the adversarial points, long double on the
  bulk).
* the walk stacks: a hierarchy exactly kFwnMaxDepth = 24 nodes deep is exact; one 25 deep is refused by svsdf_create.
* the mesh far-field bound of choiceTInit's layer 1 (prune_scale, prune_rmin): per point sdf, t*, gradient and interior
  round counts bitwise the oracle, which scans layer 1 without pruning, in the sparse and the batched schedule.
"""
import os
import sys
from fractions import Fraction

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, scenes

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
sys.path.insert(0, HERE)
sys.path.insert(0, GOLD)
import make_live_golden as mkl  # noqa: E402
import make_outer_edges_golden as mko  # noqa: E402
import test_oracle_functor_bounds as B  # noqa: E402  (meshes, polygons, point sets and the far-field restatement)

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps


def _z0(xy):
    xy = np.asarray(xy, dtype=np.float64).reshape(-1, 2)
    return np.c_[xy, np.zeros(len(xy))]


def _set_batched(monkeypatch, val):
    for var in ("SVSDF_FORCE_BATCHED", "SVSDF_FORCE_GRID_OUTER", "SVSDF_FORCE_GSIP_WIDE", "SVSDF_FORCE_GRID_GSIP"):
        monkeypatch.delenv(var, raising=False)
    if val is not None:
        monkeypatch.setenv("SVSDF_FORCE_BATCHED", val)


def _n_differ(a, b):
    a, b = np.asarray(a).reshape(len(a), -1), np.asarray(b).reshape(len(b), -1)
    return int((~((a == b) | (np.isnan(a) & np.isnan(b)))).any(axis=1).sum())


# ---------------------------------------------------------------------------------------------------------------------
# Polygon
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(B.polygons()))
def test_polygon_functor_is_bitwise_the_oracle(oracle_mod, name):
    P = B.polygons()[name]
    poly = P.reshape(-1)
    c = P.mean(axis=0)
    scale = float(np.max(np.abs(P - c)))
    rng = np.random.default_rng(2024)
    Q = np.r_[B.polygon_cases(P), _z0(c + rng.uniform(-2.0, 2.0, size=(100_000, 2)) * scale)]
    s_c = oracle_mod.shape_sdf("custom_poly", Q, polygon=poly)
    g_c = oracle_mod.shape_grad1("custom_poly", Q, polygon=poly)
    ctx = api.Context("custom_poly", polygon=poly, strict_fp=True)
    s_g, g_g = ctx.shape_sdf(Q), ctx.shape_grad1(Q)
    ctx.close()
    bad = np.flatnonzero((s_g != s_c) | (np.signbit(s_g) != np.signbit(s_c)))
    assert bad.size == 0, (name, bad.size, Q[bad[:3]], s_g[bad[:3]], s_c[bad[:3]])
    assert _n_differ(g_g, g_c) == 0, name
    # FMA build: the same function to rounding, and the same side (signbit: inside gives -dis, also -0.0 on the outline)
    ctx = api.Context("custom_poly", polygon=poly, strict_fp=False)
    s_f = ctx.shape_sdf(Q)
    ctx.close()
    tol = 1e-12 * max(1.0, float(np.abs(P).max()))
    assert np.abs(s_f - s_c).max() <= tol, (name, np.abs(s_f - s_c).max())
    assert np.array_equal(np.signbit(s_f), np.signbit(s_c)), (name, int((np.signbit(s_f) != np.signbit(s_c)).sum()))


# ---------------------------------------------------------------------------------------------------------------------
# mesh functor on every builder branch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mesh", mkl.FWN_MESHES)
def test_mesh_functor_on_every_builder_branch(oracle_mod, mesh):
    V, F, Q3 = mkl.fwn_mesh(mesh)
    m = (V, F)
    Q = _z0(Q3[:, :2])  # the planner evaluates the z = 0 plane only
    w = oracle_mod.mesh_eval(m, Q, "winding")
    d2 = oracle_mod.mesh_eval(m, Q, "sqr_distance")
    on_plane = Q3[:, 2] == 0.0
    assert on_plane.sum() >= 1000
    w_ref = np.load(os.path.join(GOLD, "ref_live.npz"))[f"fwn_{mesh}_w"]
    assert np.array_equal(w[on_plane], w_ref[on_plane])  # the reference's own code at these very points
    want = (1.0 - 2.0 * w) * np.sqrt(d2)
    ctx = api.Context("ignored", strict_fp=True, mesh=m)
    got = ctx.shape_sdf(Q)
    ctx.close()
    assert _n_differ(got, want) == 0, (mesh, _n_differ(got, want))
    for pp in ((0.0, 0.0, 0.0), (0.6, -0.3, 25.0)):
        ctx = api.Context("ignored", poly_params=pp, strict_fp=True, mesh=m)
        got = ctx.shape_sdf(Q)
        ctx.close()
        want = oracle_mod.mesh_eval(m, Q, "sdf", poly_params=pp)
        assert _n_differ(got, want) == 0, (mesh, pp, _n_differ(got, want))
    ctx = api.Context("ignored", strict_fp=False, mesh=m)
    got = ctx.shape_sdf(Q)
    ctx.close()
    ok = d2 > 0.0
    w_back = (1.0 - got[ok] / np.sqrt(d2[ok])) / 2.0
    assert np.abs(w_back - w[ok]).max() < 1e-12, (mesh, np.abs(w_back - w[ok]).max())


# ---------------------------------------------------------------------------------------------------------------------
# closest-distance pruning
# ---------------------------------------------------------------------------------------------------------------------
def _seg_d2(p, a, b, zero, clamp):
    """Squared distance from p to segment ab; array or Fraction arithmetic (clamp: min / max of the type)."""
    ab = [b[k] - a[k] for k in range(3)]
    ap = [p[k] - a[k] for k in range(3)]
    den = ab[0] * ab[0] + ab[1] * ab[1] + ab[2] * ab[2]
    num = ap[0] * ab[0] + ap[1] * ab[1] + ap[2] * ab[2]
    t = clamp(num, den)
    e = [ap[k] - t * ab[k] for k in range(3)]
    return e[0] * e[0] + e[1] * e[1] + e[2] * e[2]


def _tri_d2_exact(p, a, b, c):
    """Exact squared distance from p to triangle abc (Fractions): the plane projection if it falls inside, else the nearest
    edge.  A formulation independent of Ericson's region walk used by the kernels and the oracle."""
    def clamp(num, den):
        if den == 0:
            return Fraction(0)
        return min(max(num / den, Fraction(0)), Fraction(1))

    best = min(_seg_d2(p, a, b, 0, clamp), _seg_d2(p, b, c, 0, clamp), _seg_d2(p, c, a, 0, clamp))
    u = [b[k] - a[k] for k in range(3)]
    v = [c[k] - a[k] for k in range(3)]
    n = [u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]]
    nn = n[0] * n[0] + n[1] * n[1] + n[2] * n[2]
    if nn == 0:
        return best
    ap = [p[k] - a[k] for k in range(3)]
    h = ap[0] * n[0] + ap[1] * n[1] + ap[2] * n[2]
    x = [p[k] - h / nn * n[k] for k in range(3)]
    inside = True
    for s, e in ((a, b), (b, c), (c, a)):
        se = [e[k] - s[k] for k in range(3)]
        sx = [x[k] - s[k] for k in range(3)]
        cr = [se[1] * sx[2] - se[2] * sx[1], se[2] * sx[0] - se[0] * sx[2], se[0] * sx[1] - se[1] * sx[0]]
        if cr[0] * n[0] + cr[1] * n[1] + cr[2] * n[2] < 0:
            inside = False
    return min(best, h * h / nn) if inside else best


def _mesh_d2_longdouble(T, p):
    """Squared distance from p to every triangle of T [nf, 3, 3] in long double (same formulation, vectorised)."""
    T = T.astype(np.longdouble)
    p = np.asarray(p, dtype=np.longdouble)
    a, b, c = T[:, 0], T[:, 1], T[:, 2]

    def seg(s, e):
        se, sp = e - s, p - s
        den = (se * se).sum(axis=1)
        with np.errstate(invalid="ignore", divide="ignore"):
            t = np.where(den > 0, np.clip((sp * se).sum(axis=1) / np.where(den > 0, den, 1), 0, 1), 0)
        r = sp - t[:, None] * se
        return (r * r).sum(axis=1)

    best = np.minimum(np.minimum(seg(a, b), seg(b, c)), seg(c, a))
    n = np.cross(b - a, c - a)
    nn = (n * n).sum(axis=1)
    h = ((p - a) * n).sum(axis=1)
    ok = nn > 0
    x = p - np.where(ok, h / np.where(ok, nn, 1), 0)[:, None] * n
    inside = ok.copy()
    for s, e in ((a, b), (b, c), (c, a)):
        inside &= (np.cross(e - s, x - s) * n).sum(axis=1) >= 0
    plane = np.where(inside, h * h / np.where(ok, nn, 1), np.inf)
    return np.minimum(best, plane)


def exact_d2(V, F, Q, exact_idx):
    """min over all faces of the exact squared point-triangle distance: long double for every point, fractions.Fraction for
    the points in exact_idx (over the faces whose long-double distance is within a margin of the minimum)."""
    T = np.asarray(V, dtype=np.float64)[np.asarray(F)]
    out = np.empty(len(Q))
    Tf = None
    for i, q in enumerate(Q):
        d = _mesh_d2_longdouble(T, q)
        if i in exact_idx:
            if Tf is None:
                Tf = [[[Fraction(float(x)) for x in v] for v in t] for t in T]
            M2 = float(np.max(np.abs(T))) ** 2 + float(np.dot(q, q))
            cand = np.flatnonzero(d <= d.min() * (1 + 1e-9) + 1e-24 * (1.0 + M2))
            qf = [Fraction(float(x)) for x in q]
            out[i] = float(min(_tri_d2_exact(qf, *Tf[f]) for f in cand))
        else:
            out[i] = float(d.min())
    return out


def pruning_cases():
    """name -> (V, F, Q [m, 3], indices of Q to check with exact rationals)."""
    rng = np.random.default_rng(404)
    cases = {}
    # 1. a mesh symmetric about x = 0, y = 0 and y = +-x (vertices mirrored exactly): queries on the symmetry planes, where
    #    faces in different subtrees are at exactly the same distance
    base = [(3.0, 0.0), (1.2, 0.5), (0.5, 1.2)]
    outline = []
    for q in range(4):  # rotate by 90 degrees exactly: (x, y) -> (-y, x)
        for x, y in base:
            for _ in range(q):
                x, y = -y, x
            outline.append((x, y))
    V, F = scenes.extrude_outline(np.array(outline), half_height=0.45)
    r = np.r_[np.linspace(0.0, 6.0, 61), rng.uniform(0.0, 6.0, 200)]
    Q = np.concatenate([_z0(np.c_[r, 0 * r]), _z0(np.c_[0 * r, r]), _z0(np.c_[r, r]), _z0(np.c_[r, -r]), _z0(np.c_[-r, -r]),
                        _z0(np.c_[-r, 0 * r])])
    cases["symmetry_planes"] = (V, F, Q, set(range(0, len(Q), 7)))
    # 2. two walls in different subtrees (one at x = +3, one at x = -3 (1 + 1e-13)) with filler faces behind each: queries
    #    between them whose two candidate distances differ by ~1e-13 relative, either way round
    def wall(x0, s=1.0):
        return [[x0, -s, -0.6], [x0, s, -0.6], [x0, 0.0, 0.7]]

    tris = [wall(3.0), wall(-3.0 * (1.0 + 1e-13))]
    for k in range(6):
        tris += [wall(4.0 + 0.5 * k, 1.5), wall(-4.0 - 0.5 * k, 1.5)]
    V = np.array(tris).reshape(-1, 3)
    F = np.arange(len(V), dtype=np.int32).reshape(-1, 3)
    xs = np.r_[np.arange(-20, 21) * 0.5e-13, rng.uniform(-3e-12, 3e-12, 100)]
    ys = np.array([0.0, 0.3, -0.55, 0.9])
    Q = _z0(np.array([(x, y) for x in xs for y in ys]))
    cases["near_tie_1e-13"] = (V, F, Q, set(range(len(Q))))
    # 3. a flat mesh in the z = 0 plane (the star outline fanned from its centre) plus a slab around it: queries exactly at
    #    the vertices and on the edges (s + lam (e - s) in double), where every in-plane solid angle is 0
    o = scenes.star_outline(n_per_edge=2)
    n = len(o)
    Vf = np.r_[_z0(o), [[0.0, 0.0, 0.0]]]
    Ff = np.array([[n, i, (i + 1) % n] for i in range(n)], dtype=np.int32)
    Vs, Fs = scenes.extrude_outline(o * 1.6, half_height=0.3)
    V, F = np.r_[Vf, Vs], np.r_[Ff, Fs + len(Vf)]
    lam = np.array([0.0, 0.25, 0.5, 1.0 / 3.0, 0.9, 1.0])
    edges = [o[i] + l * (o[(i + 1) % n] - o[i]) for i in range(n) for l in lam] + [l * o[i] for i in range(n) for l in lam]
    Q = np.r_[_z0(np.array(edges)), _z0(rng.uniform(-5, 5, size=(300, 2)))]
    cases["vertices_and_edges"] = (V, F, Q, set(range(len(edges))))
    # 4. a mesh entirely above the plane, z in [0.3, 2]: dz2 > 0 in every box
    V, F = scenes.extrude_outline(scenes.star_outline(n_per_edge=3), half_height=0.85)
    V = V + np.array([0.0, 0.0, 1.15])
    Q = _z0(rng.uniform(-4.5, 4.5, size=(800, 2)))
    cases["above_plane"] = (V, F, Q, set(range(0, 800, 40)))
    # 5. coordinates near 1e5 (fwn_boxmag sets the boxes' error term), queries next to the surface
    V, F = scenes.extrude_outline(scenes.star_outline(n_per_edge=3))
    V = V + np.array([1.0e5, -1.0e5, 0.0])
    o = scenes.star_outline(n_per_edge=3)
    k = rng.integers(0, len(o), 1500)
    t = rng.uniform(0, 1, 1500)
    edge_pts = o[k] + t[:, None] * (np.roll(o, -1, axis=0)[k] - o[k])
    near = edge_pts * (1.0 + rng.uniform(-0.02, 0.02, 1500))[:, None] + np.array([1.0e5, -1.0e5])
    Q = np.r_[_z0(near), _z0(np.array([1.0e5, -1.0e5]) + rng.uniform(-4, 4, size=(500, 2)))]
    cases["coords_1e5"] = (V, F, Q, set(range(0, 2000, 50)))
    # 6. queries near 1e7
    V, F = scenes.extrude_outline(scenes.star_outline(n_per_edge=2))
    th = rng.uniform(0, 2 * np.pi, 600)
    rr = 10.0 ** rng.uniform(6.0, 7.2, 600)
    Q = _z0(np.c_[rr * np.cos(th), rr * np.sin(th)])
    cases["queries_1e7"] = (V, F, Q, set(range(0, 600, 30)))
    # 7. faces of ~1e-3 m and queries so far away (|q| ~ 1e5) that (float) q rounds by more than a face's size
    V, F = scenes.extrude_outline(scenes.star_outline(n_per_edge=2))
    V = V * 1e-3
    th = rng.uniform(0, 2 * np.pi, 600)
    rr = rng.uniform(0.9e5, 3.0e5, 600)
    Q = _z0(np.c_[rr * np.cos(th), rr * np.sin(th)])
    cases["far_rounding"] = (V, F, Q, set(range(0, 600, 30)))
    return cases


@pytest.mark.parametrize("name", list(pruning_cases()))
def test_closest_distance_is_the_plain_minimum(oracle_mod, name):
    V, F, Q, exact_idx = pruning_cases()[name]
    m = (V, F)
    want = oracle_mod.mesh_eval(m, Q, "sdf")
    w = oracle_mod.mesh_eval(m, Q, "winding")
    d2x = exact_d2(V, F, Q, exact_idx)
    ref = (1.0 - 2.0 * w) * np.sqrt(d2x)
    M = float(np.abs(V).max())
    qn = np.hypot(Q[:, 0], Q[:, 1])
    # 4 ulp, plus the double rounding of the face coordinates and of q where the distance is small next to them (points on
    # the surface): 8 eps (|q| + M) |1 - 2 w|
    tol = 4.0 * np.spacing(np.abs(ref)) + 8.0 * EPS * (qn + M) * np.abs(1.0 - 2.0 * w)
    for strict in (True, False):
        ctx = api.Context("ignored", strict_fp=strict, mesh=m)
        got = ctx.shape_sdf(Q)
        ctx.close()
        if strict:
            bad = np.flatnonzero(got != want)
            assert bad.size == 0, (name, bad.size, Q[bad[:3]], got[bad[:3]], want[bad[:3]])
        err = np.abs(got - ref)
        ulps = err[ref != 0] / np.spacing(np.abs(ref[ref != 0]))
        print(f"{name} strict={strict}: max |sdf - exact| {err.max():.3g}; {np.mean(ulps <= 4.0):.1%} of the points within 4 ulp")
        bad = np.flatnonzero(err > tol)
        assert bad.size == 0, (name, strict, bad.size, Q[bad[:3]], got[bad[:3]], ref[bad[:3]])


# ---------------------------------------------------------------------------------------------------------------------
# walk-stack limits
# ---------------------------------------------------------------------------------------------------------------------
CHAIN_RATIO, CHAIN_24, CHAIN_25 = 0.5, 104, 112


def chain_mesh(n, r=CHAIN_RATIO, size=0.3):
    """n triangles, triangle k centred at x = r^k with size ~ r^k: with r = 0.5 the builder's binned split finds more than
    15/16 of the items in its lowest bin at every level and peels the far sixteenth off, so the hierarchy deepens by one
    node per level: 104 faces give depth 24 (the deepest the device stacks hold), 112 give 25."""
    V = []
    for k in range(n):
        s = r ** k
        V += [[s, -size * s, -size * s], [s, size * s, -size * s], [s, 0.0, size * s]]
    return np.array(V), np.arange(3 * n, dtype=np.int32).reshape(n, 3)


def hierarchy_depth(ch):
    def d(node):
        best = 0
        for c in ch[node]:
            if c == B.EMPTY:
                break
            if c & B.INTERNAL:
                best = max(best, d(int(c & 0x7FFFFFFF)))
        return best + 1

    return d(0)


def test_hierarchy_of_depth_24_is_exact_and_25_is_refused(oracle_mod):
    V, F = chain_mesh(CHAIN_24)
    assert hierarchy_depth(api.mesh_fwn_host(V, F)[0]) == 24
    rng = np.random.default_rng(24)
    q = []
    for k in range(CHAIN_24):  # next to every triangle, the deepest ones most
        s = CHAIN_RATIO ** k
        per = 40 if k >= CHAIN_24 - 12 else 4
        q.append(np.c_[s + s * rng.uniform(-0.6, 0.6, per), s * rng.uniform(-0.6, 0.6, per)])
    Q = _z0(np.concatenate(q))
    want = oracle_mod.mesh_eval((V, F), Q, "sdf")
    ctx = api.Context("ignored", strict_fp=True, mesh=(V, F))
    got = ctx.shape_sdf(Q)
    ctx.close()
    assert _n_differ(got, want) == 0, _n_differ(got, want)
    V, F = chain_mesh(CHAIN_25)
    assert hierarchy_depth(api.mesh_fwn_host(V, F)[0]) == 25
    with pytest.raises(api.SvsdfError):
        api.Context("ignored", strict_fp=True, mesh=(V, F))


# ---------------------------------------------------------------------------------------------------------------------
# far-field pruning end to end
# ---------------------------------------------------------------------------------------------------------------------
def _traj(N=8):
    init_s, final_s, q, T = scenes.make_trajectory("star", N)
    b = scenes.minco_dense(init_s, final_s, q, T)
    return T, np.ascontiguousarray(b.T).reshape(-1), b


def _points_around(rng, path, n, r0, r1):
    k = rng.integers(0, len(path), n)
    th = rng.uniform(0, 2 * np.pi, n)
    r = rng.uniform(r0, r1, n)
    return _z0(path[k, :2] + np.c_[r * np.cos(th), r * np.sin(th)])


FAR_CASES = {"sdHorseshoe_obj": 400, "sdArc_obj": 200, "star_obj_x1e3": 400, "star_obj_off_origin": 400}


@pytest.mark.parametrize("name", list(FAR_CASES))
def test_far_field_pruning_end_to_end(oracle_mod, monkeypatch, name):
    V, F, pp = B.bound_cases()[name]
    Rv, rho0, omega, finite = B.far_field_bound(V, F, pp)
    assert finite and omega < B.PRUNE_OMEGA_MAX  # the pruning is on for this mesh
    T, co, b = _traj()
    path = scenes.eval_traj_xy(b, T, np.linspace(0.0, float(T.sum()), 2000))
    rng = np.random.default_rng(77)
    pts = np.r_[_points_around(rng, path, FAR_CASES[name], rho0, 3.0 * rho0), _points_around(rng, path, 30, 0.0, Rv)]
    orc = oracle_mod.Oracle(mesh=(V, F), poly_params=pp, threads=oracle_mod.num_procs())
    orc.set_traj(T, co)
    ref = orc.query(pts)
    assert (ref[3] > 0).sum() >= 3  # some points are interior: k_gsip runs
    for batched in ("0", "1"):
        _set_batched(monkeypatch, batched)
        ctx = api.Context("ignored", poly_params=pp, strict_fp=True, mesh=(V, F))
        got = ctx.query(T, co, pts)
        ctx.close()
        for a, r_, what in zip(got, ref, ("sdf", "t*", "gradient", "rounds")):
            assert _n_differ(a, r_) == 0, (name, batched, what, _n_differ(a, r_))


def test_far_field_pruning_is_active_on_a_long_trajectory(oracle_mod, monkeypatch):
    """long64's trajectory (64 pieces, D = 299.84 s: K1 = 1998 layer-1 samples) with shapes/sdHorseshoe.obj: bitwise the
    oracle's unpruned scan.  The pruning is on for this mesh (omega < 0.45, asserted by the restatement).  The executed
    evaluation counts are printed, not asserted: svsdf_executed_evals counts every lane evaluation of layers 1-4 and of the
    descents, and the descents dominate it here (about 2 900 per point in the sparse schedule, with or without the far-field
    factor), so it cannot show the layer-1 skips on its own."""
    V, F, pp = B.bound_cases()["sdHorseshoe_obj"]
    Rv, rho0, omega, finite = B.far_field_bound(V, F, pp)
    _, T, co, _ = mko.scene("long64")
    D = float(T.sum())
    K1 = int(D / 0.15)
    assert K1 >= 1000
    b = co.reshape(3, -1).T
    path = scenes.eval_traj_xy(b, T, np.linspace(0.0, D, 20000))
    pts = _points_around(np.random.default_rng(78), path, 150, rho0, 3.0 * rho0)
    orc = oracle_mod.Oracle(mesh=(V, F), threads=oracle_mod.num_procs())
    assert finite and omega < B.PRUNE_OMEGA_MAX
    orc.set_traj(T, co)
    ref = orc.query(pts)
    for batched in ("0", "1"):
        _set_batched(monkeypatch, batched)
        ctx = api.Context("ignored", strict_fp=True, mesh=(V, F))
        ctx.executed_evals(True)
        got = ctx.query(T, co, pts)
        per_point = ctx.executed_evals(False) / len(pts)
        ctx.close()
        print(f"long64 sdHorseshoe batched={batched}: {per_point:.1f} executed evaluations per point, K1 = {K1}")
        for a, r_, what in zip(got, ref, ("sdf", "t*", "gradient", "rounds")):
            assert _n_differ(a, r_) == 0, (batched, what, _n_differ(a, r_))
