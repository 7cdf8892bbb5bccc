"""GPU (-m gpu): svsdf_swept_contour_multi — every problem of a batch is its own svsdf_swept_contour call on the same context, bit for bit
in every output (grid, vertices, segments, triangles, clipped, n_evaluated, field), over shapes, pre-transforms, the mesh functor, the
scale schedule, both builds, iso, h, boxes and want_field; the outlines of two strict cases against the checker oracle/swept_oracle.hpp;
launches, non-interference and interleaving; the limits of n and of the corners, errors; plan_batch(outline=...) against
generate_traj(outline=...)."""
import os

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, plan, scenes
from oracle import swept_py

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SHAPES16 = ["star", "sdHorseshoe", "sdPie", "sdPie2", "sdArc", "sdTunnel", "sdCutDisk", "sdTrapezoid", "sdRhombus", "sdHeart",
            "sdRoundedX", "bigX", "sdRoundedCross", "sdOrientedVesica", "sdMoon", "sdUnevenCapsule"]
ISOS = [0.0, 0.7, -0.3]


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.uint64)


def traj(N, seed, dur=2.5, start=(0.0, 0.0)):
    """(T, coeffs column-major) of a seeded spline; N = 1 is a single quintic built by hand."""
    if N == 1:
        rng = np.random.default_rng(seed)
        b = np.zeros((6, 3))
        b[0] = [start[0] + rng.uniform(-2, 2), start[1] + rng.uniform(-2, 2), 0.3]
        b[1] = [1.2, 0.4, 0.2]
        b[2] = [0.05, -0.02, 0.0]
        return np.array([dur]), b.T.reshape(-1).copy()
    init_s, final_s, q, _ = scenes.make_trajectory("star", N=N, seed=seed, start=start, goal=(start[0] + 3.0 * N, start[1] + 4.0))
    T = np.full(N, dur)
    b, _, _, _ = api.minco_forward(init_s, final_s, q, T)
    return T, np.ascontiguousarray(b.T).reshape(-1)


def mixed_batch():
    """N = 1, 8, 23 and 64; short and long durations; a path far from the others; the same trajectory twice."""
    a = traj(8, 31)
    return [traj(1, 3), a, traj(23, 5, 0.4), traj(64, 7, 4.6), traj(8, 9, 0.25, start=(400.0, -300.0)), a, traj(1, 11, 12.0)]


def ctx_for(shape, pp=(0.0, 0.0, 0.0), strict=True):
    if shape == "star_obj_mesh":
        g = np.load(os.path.join(GOLD, "fwn_ref.npz"))
        return api.Context("star", poly_params=pp, strict_fp=strict, mesh=(g["star_V"], g["star_F"]))
    return api.Context(shape, poly_params=pp, strict_fp=strict)


def assert_same(m, s, what=""):
    assert (m.i0, m.j0, m.nx, m.ny, m.clipped, m.n_evaluated) == (s.i0, s.j0, s.nx, s.ny, s.clipped, s.n_evaluated), what
    assert np.array_equal(bits(m.vertices), bits(s.vertices)), what
    assert np.array_equal(m.segments, s.segments) and np.array_equal(m.triangles, s.triangles), what
    assert (m.field is None) == (s.field is None), what
    if m.field is not None:
        assert np.array_equal(bits(m.field), bits(s.field)), what  # NaN pattern and bits


def check_multi(ctx, trajs, h, iso, box=None, want_field=False):
    got = ctx.swept_contour_multi(trajs, h, iso, box=box, want_field=want_field)
    assert len(got) == len(trajs)
    for k, (T, co) in enumerate(trajs):
        assert_same(got[k], ctx.swept_contour(T, co, h, iso, box=box, want_field=want_field), (k, h, iso, box))
    return got


@pytest.mark.parametrize("shape,pp", [(s, (0.0, 0.0, 0.0)) for s in SHAPES16 + ["Circle", "Polygon"]] +
                         [("star", (0.4, -0.3, 25.0)), ("Polygon", (0.4, -0.3, 25.0))])
def test_multi_equals_single_every_shape(shape, pp):
    ctx = ctx_for(shape, pp)
    trajs = mixed_batch()
    for iso in ISOS:
        check_multi(ctx, trajs, 0.2, iso, want_field=(iso == 0.7))
    ctx.close()


@pytest.mark.parametrize("strict", [True, False])
def test_multi_equals_single_builds_and_fine_grid(strict):
    ctx = ctx_for("star", strict=strict)
    trajs = mixed_batch()
    for iso in ISOS:
        got = check_multi(ctx, trajs, 0.05, iso, want_field=True)
        assert all(len(g.triangles) > 0 for g in got) or iso < 0
    ctx.close()


def test_multi_equals_single_mesh_and_scale():
    ctx = ctx_for("star_obj_mesh")
    trajs = [traj(1, 7), traj(1, 8, 1.0), traj(2, 9, 0.5)]
    box = (-4.0, -4.0, 10.0, 6.0)  # the mesh functor has no far-field bound
    for iso in ISOS:
        check_multi(ctx, trajs, 0.25, iso, box=box, want_field=True)
    ctx.close()
    for strict in (True, False):
        ctx = ctx_for("star", strict=strict)
        ctx.set_scale(**api.EXAMPLE_SCALE)
        trajs = mixed_batch()
        for iso in ISOS:
            check_multi(ctx, trajs, 0.2, iso, want_field=True)
        ctx.close()


def test_shared_box_clips_and_empties():
    """One user box for all: it cuts some problems' regions (clipped = 1), misses the far path (nothing evaluated beside problems
    with corners) and holds no corner of others."""
    ctx = ctx_for("star")
    trajs = mixed_batch()
    box = (2.0, -1.0, 9.0, 3.0)
    for want_field in (False, True):
        for h in (0.05, 0.2):
            got = check_multi(ctx, trajs, h, 0.7, box=box, want_field=want_field)
            assert any(g.clipped for g in got) and got[4].n_evaluated == 0 and len(got[4].vertices) == 0
            assert any(g.n_evaluated > 0 for g in got)
    ctx.close()


@pytest.mark.parametrize("shape", ["star", "Polygon"])
def test_outline_is_the_checker_on_the_dense_field(shape):
    ctx = ctx_for(shape)
    trajs = mixed_batch()[:4]
    for iso in (0.0, 0.7):
        got = ctx.swept_contour_multi(trajs, 0.2, iso, want_field=True)
        for (T, co), r in zip(trajs, got):
            x, y = r.corners()
            X, Y = np.meshgrid(x, y)
            dense = ctx.query(T, co, np.c_[X.reshape(-1), Y.reshape(-1), np.zeros(X.size)], outer_only=True)[0].reshape(r.ny, r.nx)
            ev = ~np.isnan(r.field)
            assert np.array_equal(bits(r.field[ev]), bits(dense[ev])) and np.all(dense[~ev] > iso)
            o = swept_py.swept_contour(dense, r.i0, r.j0, 0.2, iso)
            assert np.array_equal(bits(r.vertices), bits(o.vertices))
            assert np.array_equal(r.segments, o.segments) and np.array_equal(r.triangles, o.triangles) and r.clipped == o.clipped
    ctx.close()


def test_launches_and_non_interference():
    ctx = ctx_for("star")
    T, co = traj(8, 31)
    rng = np.random.default_rng(3)
    pts = np.c_[rng.uniform(-2, 26, 3000), rng.uniform(-4, 8, 3000), np.zeros(3000)]
    ctx.set_points(pts)
    ctx.cost_grad(T, co)
    ref = ctx.cost_grad(T, co)  # after two evaluations (the k_gsip variant follows the previous evaluation)
    resident = ctx.get_points().copy()
    counts = []
    for n in (1, 7, 300, 0):
        n0 = ctx.kernel_launches()
        got = ctx.swept_contour_multi([(T, co)] * n, 0.2, 0.7)
        counts.append(ctx.kernel_launches() - n0)
        assert len(got) == n
    assert counts[0] == counts[1] == counts[2] > 0 and counts[3] == 0, counts
    # a box that holds no needed corner: none of the evaluation's launches
    n0 = ctx.kernel_launches()
    got = ctx.swept_contour_multi([(T, co)] * 5, 0.2, 0.7, box=(500.0, 500.0, 501.0, 501.0))
    assert all(g.n_evaluated == 0 for g in got) and ctx.kernel_launches() - n0 < counts[0]
    after = ctx.cost_grad(T, co)
    for x, y in zip(ref, after):
        assert np.array_equal(bits(x), bits(y))
    assert np.array_equal(bits(resident), bits(ctx.get_points()))
    ctx.close()


def test_interleaved_calls_equal_a_fresh_context():
    ctx = ctx_for("star")
    pool = mixed_batch()
    fresh = ctx_for("star")
    want = [fresh.swept_contour(T, co, 0.2, 0.7, want_field=True) for T, co in pool]
    fresh.close()
    for n in (7, 300, 1, 50):
        idx = [k % len(pool) for k in range(n)]
        got = ctx.swept_contour_multi([pool[k] for k in idx], 0.2, 0.7, want_field=True)
        for k, g in zip(idx, got):
            assert_same(g, want[k], (n, k))
        k = n % len(pool)
        assert_same(ctx.swept_contour(*pool[k], 0.2, 0.7, want_field=True), want[k], ("single", n))
    ctx.close()


def test_most_problems_and_one_more():
    ctx = ctx_for("star")
    pool = [traj(1, s) for s in range(5)]
    box = (-0.3, -0.3, 0.3, 0.3)
    n = 65535
    trajs = [pool[k % len(pool)] for k in range(n)]
    got = ctx.swept_contour_multi(trajs, 0.1, 0.7, box=box)
    assert len(got) == n
    for k in (0, 1, 2, 3, 4, 1234, 40000, n - 1):
        assert_same(got[k], ctx.swept_contour(*trajs[k], 0.1, 0.7, box=box), k)
    assert any(got[k].n_evaluated > 0 for k in range(5))
    with pytest.raises(api.SvsdfError) as e:
        ctx.swept_contour_multi(trajs + [pool[0]], 0.1, 0.7, box=box)
    assert "status -1" in str(e.value)
    ctx.close()


def test_corner_total_over_int32_is_refused():
    """Nine problems of about 2^28 corners each (a 16001 x 16001 box at h = 1e-3, under max_corners = 2^28) hold more than 2^31 - 1
    corners: refused before anything is allocated (they would need about 48 GB of device memory)."""
    ctx = ctx_for("star")
    T, co = traj(1, 3)
    h = 1e-3
    box = (0.0, 0.0, 16000 * h, 16000 * h)
    assert ctx.swept_contour(T, co, 0.1, box=box).nx == 161  # the box itself is valid
    with pytest.raises(api.SvsdfError) as e:
        ctx.swept_contour_multi([(T, co)] * 9, h, 0.0, box=box, max_corners=1 << 28)
    assert "status -1" in str(e.value) and "2^31 - 1 corners" in str(e.value)
    got = ctx.swept_contour_multi([(T, co)] * 3, 0.1, 0.0)  # the context still works
    assert_same(got[2], ctx.swept_contour(T, co, 0.1, 0.0))
    ctx.close()


def test_errors():
    ctx = ctx_for("star")
    T, co = traj(2, 5)
    good = [traj(1, 3), (T, co)]
    for kw in (dict(h=0.0), dict(h=-1.0), dict(h=np.nan), dict(h=np.inf), dict(h=0.1, iso=np.nan), dict(h=0.1, iso=np.inf),
               dict(h=0.1, box=(1.0, 0.0, 0.0, 1.0)), dict(h=0.1, box=(0.0, 1.0, 1.0, 0.0)), dict(h=0.1, box=(0.0, 0.0, np.nan, 1.0)),
               dict(h=1e-4, box=(0.0, 0.0, 10.0, 10.0)), dict(h=0.1, max_corners=(1 << 28) + 1), dict(h=0.1, max_corners=3),
               dict(h=1e-3, max_corners=1000)):
        with pytest.raises(api.SvsdfError) as e:
            ctx.swept_contour_multi(good, **kw)
        assert "status -1" in str(e.value), kw
    for bad in ((np.array([1.0, -1.0]), co), (np.array([1.0, np.nan]), co), (np.array([200.0, 200.0]), co),
                (T, np.where(np.arange(co.size) == 3, np.nan, co)), (np.zeros(65), np.zeros(18 * 65))):
        n0 = ctx.kernel_launches()
        with pytest.raises(api.SvsdfError) as e:
            ctx.swept_contour_multi(good + [bad] + good, 0.1)
        assert "status -1" in str(e.value) and ctx.kernel_launches() == n0
    assert ctx.swept_contour_multi([], 0.1) == []
    ctx.close()
    # a shape without a far-field bound: a mesh with a vertex at 1e160 (the squares of its radius overflow, so svsdf_create keeps no
    # bound; tests/test_oracle_functor_bounds.py restates that rule)
    V = np.array([[-3.0, -2.0, -0.4], [1e160, -1.0, 0.3], [0.5, 3.5, 0.8]])
    mesh = api.Context("star", mesh=(V, np.array([[0, 1, 2]], dtype=np.int32)))
    n0 = mesh.kernel_launches()
    for call in (lambda: mesh.swept_contour_multi(good, 0.25), lambda: mesh.swept_contour(*good[0], 0.25)):
        with pytest.raises(api.SvsdfError) as e:
            call()
        assert "status -1" in str(e.value) and "far-field bound" in str(e.value)
    assert mesh.kernel_launches() == n0
    mesh.close()
    # a non-finite field value (the single call's construction: a path at x ~ 1.7e308) among good problems
    ctx = ctx_for("star")
    b = np.zeros((6, 3))
    b[0, 0] = b[5, 0] = 1.7e308
    far = (np.array([1.0]), b.T.reshape(-1).copy())
    box = (-2.0, -2.0, 2.0, 2.0)
    got = ctx.swept_contour_multi([good[0], far, good[1]], 0.5, box=box, want_field=True)
    assert isinstance(got[1], api.SvsdfError) and "status -4" in str(got[1])
    for k in (0, 2):
        assert_same(got[k], ctx.swept_contour(*good[k // 2], 0.5, box=box, want_field=True), k)
    ctx.close()


@pytest.fixture(scope="module")
def star_scene():
    g = np.load(os.path.join(GOLD, "map_star_pcd.npz"))
    res, ks = float(g["occupancy_resolution"]), int(g["kernel_size"])
    cmap = plan.gridmap3d_from_cloud(g["points"], res, int(g["sta_threshold"]))
    free = np.argwhere(~cmap.occ.any(axis=2))
    pick = free[np.random.default_rng(7).choice(len(free), size=(11, 2), replace=False)]
    xy = cmap.boundary_min[:2] + (pick + 0.5) * cmap.res
    kw = dict(kernel_size=ks, traj_parlength=float(g["traj_parlength"]))
    return cmap, kw, np.r_[[g["start"][:2]], xy[:, 0]], np.r_[[g["end"][:2]], xy[:, 1]]


def ctx_new():
    return api.Context("star", weight_p=scenes.YAML["weight_p"], safety_hor=scenes.YAML["safety_hor"], rho=scenes.YAML["rho"])


@pytest.mark.parametrize("n,repair", [(12, 0), (4, 1)])
def test_plan_batch_outline_equals_generate_traj(star_scene, n, repair):
    cmap, kw, st, go = star_scene
    outline = dict(h=0.1, iso=scenes.YAML["safety_hor"])
    stats = {}
    got = plan.plan_batch(ctx_new(), cmap, st[:n], go[:n], outline=outline, repair=repair, stats=stats, **kw)
    assert stats["outline_s"] > 0.0
    with_outline = 0
    for q in range(n):
        r = plan.generate_traj(ctx_new(), cmap, st[q], go[q], outline=outline, repair=repair, **kw)
        b = got[q]
        assert ("outline" in b) == ("outline" in r) == ("T" in r), q
        if "outline" in r:
            with_outline += 1
            assert np.array_equal(bits(b["T"]), bits(r["T"])) and np.array_equal(bits(b["coeffs"]), bits(r["coeffs"]))
            assert_same(b["outline"], r["outline"], q)
            assert b["outline"].clipped == 0 and len(b["outline"].triangles) > 0
    assert with_outline >= 2


def test_outline_none_is_today(star_scene):
    cmap, kw, st, go = star_scene
    a = plan.plan_batch(ctx_new(), cmap, st[:4], go[:4], **kw)
    b = plan.plan_batch(ctx_new(), cmap, st[:4], go[:4], outline=None, **kw)
    for x, y in zip(a, b):
        assert x.keys() == y.keys() and "outline" not in y
        for key in ("T", "coeffs", "x"):
            if key in x:
                assert np.array_equal(bits(x[key]), bits(y[key]))
    r0 = plan.generate_traj(ctx_new(), cmap, st[0], go[0], **kw)
    r1 = plan.generate_traj(ctx_new(), cmap, st[0], go[0], outline=None, **kw)
    assert r0.keys() == r1.keys() and "outline" not in r1
    assert np.array_equal(bits(r0["coeffs"]), bits(r1["coeffs"]))
