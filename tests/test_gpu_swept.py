"""GPU (-m gpu): svsdf_swept_contour — the narrow-band mesher against the dense alternative (svsdf_query(outer_only) on every corner of
the same grid, contoured by the CPU checker oracle/swept_oracle.hpp), bit for bit, over shapes, pre-transforms, the mesh functor, the
scale schedule, both builds and N = 1 .. 64; geometry, boxes, non-interference, determinism, launches and errors."""
import os

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, plan, scenes
from oracle import oracle_py, swept_py

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SHAPES16 = ["star", "sdHorseshoe", "sdPie", "sdPie2", "sdArc", "sdTunnel", "sdCutDisk", "sdTrapezoid", "sdRhombus", "sdHeart",
            "sdRoundedX", "bigX", "sdRoundedCross", "sdOrientedVesica", "sdMoon", "sdUnevenCapsule"]


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.uint64)


def traj(N, seed, dur=2.5):
    """(T, coeffs column-major) of a seeded spline; N = 1 is a single quintic built by hand."""
    if N == 1:
        rng = np.random.default_rng(seed)
        b = np.zeros((6, 3))
        b[0] = [rng.uniform(-2, 2), rng.uniform(-2, 2), 0.3]
        b[1] = [1.2, 0.4, 0.2]
        b[2] = [0.05, -0.02, 0.0]
        return np.array([dur]), b.T.reshape(-1).copy()
    init_s, final_s, q, _ = scenes.make_trajectory("star", N=N, seed=seed, start=(0.0, 0.0), goal=(3.0 * N, 4.0))
    T = np.full(N, dur)
    b, _, _, _ = api.minco_forward(init_s, final_s, q, T)
    return T, np.ascontiguousarray(b.T).reshape(-1)


def line(L, dur, yaw=0.3):
    """Straight, constant-yaw path of length L along x."""
    b = np.zeros((6, 3))
    b[0, 2] = yaw
    b[1, 0] = L / dur
    return np.array([dur]), b.T.reshape(-1).copy()


def ctx_for(shape, pp=(0.0, 0.0, 0.0), strict=True):
    if shape == "star_obj_mesh":
        g = np.load(os.path.join(GOLD, "fwn_ref.npz"))
        return api.Context("star", poly_params=pp, strict_fp=strict, mesh=(g["star_V"], g["star_F"]))
    return api.Context(shape, poly_params=pp, strict_fp=strict)


def grid_xy(r):
    x, y = r.corners()
    X, Y = np.meshgrid(x, y)
    return np.c_[X.reshape(-1), Y.reshape(-1), np.zeros(X.size)]


def check_band_against_dense(ctx, T, co, h, iso, box=None):
    """The band result equals the checker on the dense field, every evaluated corner is svsdf_query's value, every skipped corner > iso."""
    r = ctx.swept_contour(T, co, h, iso, box=box, want_field=True)
    dense = ctx.query(T, co, grid_xy(r), outer_only=True)[0].reshape(r.ny, r.nx)
    ev = ~np.isnan(r.field)
    assert r.n_evaluated == int(ev.sum()) > 0
    assert np.array_equal(bits(r.field[ev]), bits(dense[ev]))
    assert np.all(dense[~ev] > iso), (iso, dense[~ev].min())
    o = swept_py.swept_contour(dense, r.i0, r.j0, h, iso)
    assert np.array_equal(bits(r.vertices), bits(o.vertices))
    assert np.array_equal(r.segments, o.segments) and np.array_equal(r.triangles, o.triangles)
    assert r.clipped == o.clipped
    if box is None:
        assert r.clipped == 0
    return r


def h_for(ctx, T, co, corners=40000):
    r = ctx.swept_contour(T, co, 1.0)
    return max(0.02, float(np.sqrt(r.nx * r.ny / corners)))


ISOS = [0.0, 0.7, -0.3]


@pytest.mark.parametrize("shape,pp", [(s, (0.0, 0.0, 0.0)) for s in SHAPES16 + ["Circle", "Polygon"]] +
                         [("star", (0.4, -0.3, 25.0)), ("Circle", (0.2, 0.1, 10.0)), ("sdHeart", (-0.5, 0.2, -40.0))])
def test_band_equals_dense_every_shape(shape, pp):
    ctx = ctx_for(shape, pp)
    T, co = traj(8, 31)
    h = h_for(ctx, T, co)
    for iso in ISOS:
        r = check_band_against_dense(ctx, T, co, h, iso)
        if iso == 0.7:
            assert len(r.triangles) > 0 and r.n_evaluated < r.nx * r.ny
    ctx.close()


@pytest.mark.parametrize("N,dur", [(1, 2.5), (8, 2.5), (64, 4.6)])
@pytest.mark.parametrize("strict", [True, False])
def test_band_equals_dense_pieces_and_builds(N, dur, strict):
    ctx = ctx_for("star", strict=strict)
    T, co = traj(N, 40 + N, dur)
    h = h_for(ctx, T, co)
    for iso in ISOS:
        check_band_against_dense(ctx, T, co, h, iso)
    ctx.close()


def test_band_equals_dense_mesh_and_scale():
    ctx = ctx_for("star_obj_mesh")
    T, co = traj(1, 7)
    for iso in ISOS:
        check_band_against_dense(ctx, T, co, 0.25, iso)
    ctx.close()
    for strict in (True, False):
        ctx = ctx_for("star", strict=strict)
        ctx.set_scale(**api.EXAMPLE_SCALE)
        T, co = traj(8, 33)
        h = h_for(ctx, T, co)
        for iso in ISOS:
            check_band_against_dense(ctx, T, co, h, iso)
        ctx.close()


def test_band_bound_is_tight_enough_to_matter():
    """Scenes where a weaker bound shows: a static Polygon (the bar's tips lie 0.05 inside its radius bound) on a fine grid, and a
    fast Circle whose samples lie about 1.4 m apart (the path between them is covered only through delta_k)."""
    ctx = ctx_for("Polygon")
    T = np.array([1.0])
    co = np.zeros(18)
    for iso in ISOS:
        check_band_against_dense(ctx, T, co, 0.02, iso)
    ctx.close()
    ctx = ctx_for("Circle")
    T, co = line(20.0, 2.0)
    for iso in ISOS:
        check_band_against_dense(ctx, T, co, 0.05, iso)
    ctx.close()


@pytest.mark.parametrize("shape", ["star", "Circle"])
def test_strict_field_is_the_oracle_end_to_end(shape):
    ctx = ctx_for(shape)
    orc = oracle_py.Oracle(shape, threads=min(8, oracle_py.num_procs()))
    T, co = traj(2, 5)
    orc.set_traj(T, co)
    for iso in (0.0, 0.7):
        r = ctx.swept_contour(T, co, 0.1, iso, want_field=True)
        ev = ~np.isnan(r.field)
        pts = grid_xy(r)
        dense = orc.query_outer(pts)[0].reshape(r.ny, r.nx)
        assert np.array_equal(bits(r.field[ev]), bits(dense[ev]))
        o = swept_py.swept_contour(dense, r.i0, r.j0, r.h, iso)
        assert np.array_equal(bits(r.vertices), bits(o.vertices))
        assert np.array_equal(r.segments, o.segments) and np.array_equal(r.triangles, o.triangles)
    ctx.close()


def test_geometry_circle_on_a_line_and_a_resting_star():
    ctx = ctx_for("Circle")  # radius 1
    L = 6.0
    T, co = line(L, 3.0)
    for h in (0.04, 0.02):
        r = ctx.swept_contour(T, co, h)
        assert abs(r.area() - (2.0 * L + np.pi)) < 6.0 * h * (2.0 * L + 2.0 * np.pi) * h + 3 * h, (h, r.area())
        assert all(l[0] == l[-1] for l in r.loops()) and len(r.loops()) == 1
    ctx.close()
    ctx = ctx_for("star")
    b = np.zeros((6, 3))
    b[0] = [1.5, -0.7, 0.4]
    co = b.T.reshape(-1).copy()
    r = ctx.swept_contour(np.array([1.0]), co, 0.02)
    c, s = np.cos(0.4), np.sin(0.4)
    d = r.vertices[np.unique(r.segments)] - [1.5, -0.7]
    rel = np.c_[c * d[:, 0] + s * d[:, 1], -s * d[:, 0] + c * d[:, 1], np.zeros(len(d))]
    assert np.max(np.abs(ctx.shape_sdf(rel))) < 2 * 0.02
    ctx.close()


def test_boxes_clipping_and_restriction():
    ctx = ctx_for("star")
    T, co = traj(8, 31)
    r = ctx.swept_contour(T, co, 0.1, 0.0, want_field=True)
    assert r.clipped == 0
    x, y = r.corners()
    box = (x[r.nx // 3], y[r.ny // 4], x[2 * r.nx // 3], y[3 * r.ny // 4])  # cuts the swept region
    b = check_band_against_dense(ctx, T, co, 0.1, 0.0, box=box)
    assert b.clipped == 1
    # same lattice: the user box's corners are corners of the automatic box, with the same values where both evaluated them
    a0, b0 = b.i0 - r.i0, b.j0 - r.j0
    sub = r.field[b0:b0 + b.ny, a0:a0 + b.nx]
    both = ~np.isnan(sub) & ~np.isnan(b.field)
    assert np.array_equal(bits(sub[both]), bits(b.field[both]))
    ctx.close()


def test_star_scene_plan_prism_and_points(tmp_path):
    g = np.load(os.path.join(GOLD, "map_star_pcd.npz"))
    res, ks = float(g["occupancy_resolution"]), int(g["kernel_size"])
    cmap = plan.gridmap3d_from_cloud(g["points"], res, int(g["sta_threshold"]))
    ctx = api.Context("star", weight_p=scenes.YAML["weight_p"], safety_hor=scenes.YAML["safety_hor"], rho=scenes.YAML["rho"])
    p = plan.generate_traj(ctx, cmap, g["start"][:2], g["end"][:2], kernel_size=ks, traj_parlength=float(g["traj_parlength"]))
    assert p["ok"]
    T, co = p["T"], np.asarray(p["coeffs"]).reshape(-1)
    iso = scenes.YAML["safety_hor"]
    r = ctx.swept_contour(T, co, 0.05, iso)
    assert r.clipped == 0 and len(r.triangles) > 0
    path = tmp_path / "swept.obj"
    api.write_prism_obj(str(path), r, 0.0, 1.0)
    faces = [tuple(int(w) - 1 for w in ln.split()[1:]) for ln in open(path) if ln.startswith("f ")]
    edges = {}
    for t in faces:
        for k in range(3):
            e = (t[k], t[(k + 1) % 3])
            edges[e] = edges.get(e, 0) + 1
    assert all(v == 1 for v in edges.values()) and all((b, a) in edges for a, b in edges)
    # every query point with f <= iso lies inside the outline (even-odd over all loops)
    pts = ctx.get_points()
    f = ctx.query(T, co, np.c_[pts, np.zeros(len(pts))], outer_only=True)[0]
    V = r.vertices
    P = V[r.segments[:, 0]], V[r.segments[:, 1]]
    for q in pts[f <= iso]:
        a, b = P
        cross = ((a[:, 1] > q[1]) != (b[:, 1] > q[1])) & (q[0] < a[:, 0] + (q[1] - a[:, 1]) * (b[:, 0] - a[:, 0]) / (b[:, 1] - a[:, 1] + 1e-300))
        assert np.count_nonzero(cross) % 2 == 1, q
    ctx.close()


def test_non_interference_determinism_and_launches():
    ctx = ctx_for("star")
    T, co = traj(8, 31)
    rng = np.random.default_rng(3)
    pts = np.c_[rng.uniform(-2, 26, 3000), rng.uniform(-4, 8, 3000), np.zeros(3000)]
    ctx.set_points(pts)
    before = ctx.cost_grad(T, co)
    ctx.cost_grad(T, co)
    ref = ctx.cost_grad(T, co)  # after two evaluations (the k_gsip variant follows the previous evaluation)
    n0 = ctx.kernel_launches()
    r1 = ctx.swept_contour(T, co, 0.05, 0.7, want_field=True)
    n1 = ctx.kernel_launches()
    r2 = ctx.swept_contour(T, co, 0.05, 0.7, want_field=True)
    n2 = ctx.kernel_launches()
    r3 = ctx.swept_contour(T, co, 0.2, 0.7)
    n3 = ctx.kernel_launches()
    after = ctx.cost_grad(T, co)
    for x, y in zip(ref, after):
        assert np.array_equal(bits(x), bits(y))
    assert np.array_equal(bits(before[0]), bits(after[0]))
    for a in ("vertices", "field"):
        assert np.array_equal(bits(getattr(r1, a)), bits(getattr(r2, a)))
    assert np.array_equal(r1.segments, r2.segments) and np.array_equal(r1.triangles, r2.triangles)
    assert n1 - n0 == n2 - n1 == n3 - n2 == 10  # classify, scan, compact, pose table, k_outer, scatter, count, scan, vertices, cells
    assert r3.nx * r3.ny < r1.nx * r1.ny
    ctx.close()


def test_errors():
    ctx = ctx_for("star")
    T, co = traj(2, 5)
    for kw in (dict(h=0.0), dict(h=-1.0), dict(h=np.nan), dict(h=np.inf), dict(h=0.1, iso=np.nan), dict(h=0.1, iso=np.inf),
               dict(h=0.1, box=(1.0, 0.0, 0.0, 1.0)), dict(h=0.1, box=(0.0, 1.0, 1.0, 0.0)), dict(h=0.1, box=(0.0, 0.0, np.nan, 1.0)),
               dict(h=1e-4, box=(0.0, 0.0, 10.0, 10.0)), dict(h=0.1, max_corners=(1 << 28) + 1), dict(h=1e-3, max_corners=1000)):
        with pytest.raises(api.SvsdfError) as e:
            ctx.swept_contour(T, co, **kw)
        assert "status -1" in str(e.value), kw
    for bad in ((np.array([1.0, -1.0]), co), (np.array([1.0, np.nan]), co), (np.array([200.0, 200.0]), co),
                (T, np.where(np.arange(co.size) == 3, np.nan, co))):
        with pytest.raises(api.SvsdfError):
            ctx.swept_contour(*bad, 0.1)
    # a non-finite field value: a path at x ~ 1.7e308 (the shape functor's squares overflow at every sample); its unbounded velocity
    # bound leaves no corner of the box provably outside, so all of them are evaluated
    b = np.zeros((6, 3))
    b[0, 0] = b[5, 0] = 1.7e308
    with pytest.raises(api.SvsdfError) as e:
        ctx.swept_contour(np.array([1.0]), b.T.reshape(-1).copy(), 0.5, box=(-2.0, -2.0, 2.0, 2.0))
    assert "status -4" in str(e.value)
    ctx.close()
