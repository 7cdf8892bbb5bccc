"""GPU (-m gpu): svsdf_map_clearance — the band result against the dense alternative (svsdf_query(outer_only = 0) on the centre of every
occupied column, filtered at d_max by oracle/clearance_oracle.py), bit for bit, over shapes, pre-transforms, the mesh functor, the scale
schedule, both builds, N = 1 .. 64, d_max = 0 / safety_hor / 3 / +inf and 2-D and 3-D maps; the strict build against the CPU oracle; a
scene where the band bound decides; non-interference, determinism, launches, errors; certified plans."""
import math
import os

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, plan, scenes
from oracle import clearance_oracle, oracle_py

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SHAPES16 = ["star", "sdHorseshoe", "sdPie", "sdPie2", "sdArc", "sdTunnel", "sdCutDisk", "sdTrapezoid", "sdRhombus", "sdHeart",
            "sdRoundedX", "bigX", "sdRoundedCross", "sdOrientedVesica", "sdMoon", "sdUnevenCapsule"]
KS = 17
D_MAX = [0.0, 0.7, 3.0, math.inf]


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
    b = np.zeros((6, 3))
    b[0, 2] = yaw
    b[1, 0] = L / dur
    return np.array([dur]), b.T.reshape(-1).copy()


def ctx_for(shape, pp=(0.0, 0.0, 0.0), strict=True):
    if shape == "star_obj_mesh":
        g = np.load(os.path.join(GOLD, "fwn_ref.npz"))
        return api.Context("star", poly_params=pp, strict_fp=strict, mesh=(g["star_V"], g["star_F"]))
    return api.Context(shape, poly_params=pp, strict_fp=strict)


def path_xy(T, co):
    N = len(T)
    c = np.asarray(co).reshape(3, 6 * N)
    out = []
    for i in range(N):
        t = np.linspace(0.0, T[i], 40)
        tp = t[:, None] ** np.arange(6)
        out.append(np.c_[tp @ c[0, 6 * i:6 * i + 6], tp @ c[1, 6 * i:6 * i + 6]])
    return np.concatenate(out)


def pack2d(occ, ks=KS, pad=True):
    """generateMapKernel2D layout ([(X + 2h)][ceil((Y + 2h) / 8)] bytes, y bits MSB first).  pad=True also sets the padding bits: the
    padding is not an obstacle, and must not show."""
    h = (ks - 1) // 2
    X, Y = occ.shape
    b = np.zeros((X + 2 * h, 8 * ((Y + 2 * h + 7) // 8)), dtype=np.uint8)
    if pad:
        b[:, :Y + 2 * h] = 1
    b[h:h + X, h:h + Y] = occ
    return np.packbits(b, axis=1)


def set_map(ctx, occ, origin, res):
    if occ.ndim == 2:
        ctx.set_map(pack2d(occ), occ.shape[0], occ.shape[1], KS, origin, res)
    else:
        ctx.set_map3d(plan.pack_map_kernel3d(occ, KS), *occ.shape, KS, (origin[0], origin[1], 0.0), res)


def scene_map(T, co, seed, margin=10.0, cells=20000, density=0.04, Z=1):
    """A random map around the path: (occ [X, Y(, Z)], origin, res), about `cells` columns."""
    p = path_xy(T, co)
    lo, hi = p.min(axis=0) - margin, p.max(axis=0) + margin
    res = float(np.sqrt(np.prod(hi - lo) / cells))
    X, Y = (int(v) for v in np.ceil((hi - lo) / res))
    rng = np.random.default_rng(seed)
    occ = rng.random((X, Y, Z)) < density / Z
    return (occ[:, :, 0] if Z == 1 else occ), (float(lo[0]), float(lo[1])), res


def dense_values(ctx, T, co, occ, origin, res):
    ij = clearance_oracle.occupied_columns(occ)
    xy = clearance_oracle.centres(ij, origin, res)
    sdf, ts, _, _ = ctx.query(T, co, np.c_[xy, np.zeros(len(xy))], outer_only=False)
    return ij, xy, sdf, ts


def assert_same(r, d):
    assert np.array_equal(r.ij, d["ij"])
    assert np.array_equal(bits(r.xy), bits(d["xy"]))
    assert np.array_equal(bits(r.sdf), bits(d["sdf"])) and np.array_equal(bits(r.tstar), bits(d["tstar"]))
    assert (r.n_occupied, r.n_within, r.n_colliding, r.argmin) == (d["n_occupied"], d["n_within"], d["n_colliding"], d["argmin"])
    assert bits(r.min_sdf) == bits(d["min_sdf"])


def check(ctx, T, co, occ, origin, res, d_maxes=D_MAX):
    """map_clearance equals the dense list at every d_max; returns the results."""
    set_map(ctx, occ, origin, res)
    ij, xy, sdf, ts = dense_values(ctx, T, co, occ, origin, res)
    out = []
    for d_max in d_maxes:
        r = ctx.map_clearance(T, co, d_max)
        assert_same(r, clearance_oracle.summarise(ij, xy, sdf, ts, d_max, len(ij)))
        assert r.n_within <= r.n_evaluated <= r.n_occupied
        if d_max == math.inf:
            assert r.n_evaluated == r.n_occupied
        out.append(r)
    return out


@pytest.mark.parametrize("shape,pp", [(s, (0.0, 0.0, 0.0)) for s in SHAPES16 + ["Circle", "Polygon"]] +
                         [("star", (0.4, -0.3, 25.0)), ("Circle", (0.2, 0.1, 10.0)), ("sdHeart", (-0.5, 0.2, -40.0))])
def test_band_equals_dense_every_shape(shape, pp):
    ctx = ctx_for(shape, pp)
    T, co = traj(8, 31)
    occ, origin, res = scene_map(T, co, 5)
    rs = check(ctx, T, co, occ, origin, res)
    assert rs[1].n_evaluated < rs[1].n_occupied and rs[3].n_within == rs[3].n_occupied
    ctx.close()


@pytest.mark.parametrize("N,dur", [(1, 2.5), (8, 2.5), (64, 4.6)])
@pytest.mark.parametrize("strict", [True, False])
def test_band_equals_dense_pieces_builds_and_3d(N, dur, strict):
    ctx = ctx_for("star", strict=strict)
    T, co = traj(N, 40 + N, dur)
    for Z in (1, 3):
        occ, origin, res = scene_map(T, co, 100 + N + Z, cells=40000 if N == 64 else 20000, Z=Z)
        rs = check(ctx, T, co, occ, origin, res)
        assert rs[0].n_colliding > 0 or N == 1
    ctx.close()


def test_band_equals_dense_mesh_and_scale():
    ctx = ctx_for("star_obj_mesh")
    T, co = traj(1, 7)
    occ, origin, res = scene_map(T, co, 9, cells=6000)
    check(ctx, T, co, occ, origin, res)
    ctx.close()
    for strict in (True, False):
        ctx = ctx_for("star", strict=strict)
        ctx.set_scale(**api.EXAMPLE_SCALE)
        T, co = traj(8, 33)
        occ, origin, res = scene_map(T, co, 10, Z=2)
        check(ctx, T, co, occ, origin, res)
        ctx.close()


def test_band_bound_is_tight_enough_to_matter():
    """Every cell occupied on fine grids, so that obstacles lie just inside and just outside d_max wherever the bound cuts: a static
    Polygon (the 12 m bar's tips lie 0.05 inside its radius bound), and a fast Circle whose samples lie about 1.4 m apart (the path
    between them is covered only through delta_k; a free corridor along it)."""
    ctx = ctx_for("Polygon")
    T, co = np.array([1.0]), np.zeros(18)
    res = 0.04
    occ = np.ones((400, 400), dtype=bool)
    # d_max = 0.67: the centres (6.66, +-0.02) have value 0.66 and lie 0.007 inside the radius bound 6.05 + 0.67 (1 % less misses them)
    for r in check(ctx, T, co, occ, (-8.0, -8.0), res, [0.0, 0.7, 0.05, 0.67]):
        assert r.n_evaluated < r.n_occupied and r.n_within > 0
    ctx.close()
    ctx = ctx_for("Circle")
    T, co = line(20.0, 2.0)
    res = 0.05
    occ = np.ones((520, 200), dtype=bool)
    occ[:, 95:105] = False
    for r in check(ctx, T, co, occ, (-3.0, -5.0), res, [0.0, 0.7, 0.05]):
        assert r.n_evaluated < r.n_occupied and r.n_within > 0
    ctx.close()


@pytest.mark.parametrize("shape", ["star", "Circle"])
def test_strict_values_are_the_oracle_and_centres_the_extraction(shape):
    ctx = ctx_for(shape)
    orc = oracle_py.Oracle(shape, threads=min(8, oracle_py.num_procs()))
    T, co = traj(2, 5)
    orc.set_traj(T, co)
    occ, origin, res = scene_map(T, co, 21, margin=4.0, cells=3000, density=0.08)
    occ[-1, -1] = False  # extract_points skips the cell around (999, 999) (the reference's tmp_pos): keep it free
    set_map(ctx, occ, origin, res)
    for d_max in (0.0, 0.7, math.inf):
        r = ctx.map_clearance(T, co, d_max)
        assert_same(r, clearance_oracle.clearance(orc, occ, origin, res, d_max))
    # the centres are the back end's query points: extraction with one box over the whole map
    X, Y = occ.shape
    mid = np.array([[origin[0] + 0.5 * X * res, origin[1] + 0.5 * Y * res]])
    ctx.extract_points(mid, 0.5 * max(X, Y) * res + 1.0)
    pts = ctx.get_points()
    r = ctx.map_clearance(T, co)
    assert len(pts) == r.n_occupied and np.array_equal(bits(pts), bits(r.xy))
    ctx.close()


def test_non_interference_determinism_launches_and_manager():
    ctx = ctx_for("star")
    T, co = traj(8, 31)
    rng = np.random.default_rng(3)
    pts = np.c_[rng.uniform(-2, 26, 3000), rng.uniform(-4, 8, 3000), np.zeros(3000)]
    ctx.set_points(pts)
    before = ctx.cost_grad(T, co)
    ctx.cost_grad(T, co)
    ref = ctx.cost_grad(T, co)  # after two evaluations (the k_gsip variant follows the previous evaluation)
    small = scene_map(T, co, 1, margin=4.0, cells=3000)
    large = scene_map(T, co, 2, margin=60.0, cells=2_000_000, density=0.01)
    launches, res = [], []
    for occ, origin, rs in (small, large, large):
        set_map(ctx, occ, origin, rs)
        n0 = ctx.kernel_launches()
        res.append(ctx.map_clearance(T, co, 0.7))
        launches.append(ctx.kernel_launches() - n0)
    after = ctx.cost_grad(T, co)
    for x, y in zip(ref, after):
        assert np.array_equal(bits(x), bits(y))
    assert np.array_equal(bits(before[0]), bits(after[0]))
    assert launches == [7, 7, 7]  # count, scan, write, pose table, k_outer, k_compact, k_gsip
    a, b = res[1], res[2]
    assert np.array_equal(a.ij, b.ij) and np.array_equal(bits(a.sdf), bits(b.sdf)) and np.array_equal(bits(a.tstar), bits(b.tstar))
    assert a.n_evaluated < a.n_occupied // 10
    m = api.SweptVolumeManager(ctx)
    m.updateTraj(T, co)
    assert bits(m.getMinSVSDF()) == bits(ctx.map_clearance(T, co).min_sdf)
    assert bits(m.getMinSVSDF(0.7)) == bits(b.min_sdf)
    ctx.close()


def test_errors():
    ctx = ctx_for("star")
    T, co = traj(2, 5)
    with pytest.raises(api.SvsdfError) as e:
        ctx.map_clearance(T, co)
    assert "status -3" in str(e.value)  # no map
    occ, origin, res = scene_map(T, co, 4, margin=3.0, cells=2000)
    set_map(ctx, occ, origin, res)
    for d in (-1e-9, -1.0, math.nan, -math.inf):
        with pytest.raises(api.SvsdfError) as e:
            ctx.map_clearance(T, co, d)
        assert "status -1" in str(e.value), d
    for bad in ((np.array([1.0, -1.0]), co), (np.array([1.0, np.nan]), co), (np.array([200.0, 200.0]), co),
                (T, np.where(np.arange(co.size) == 3, np.nan, co))):
        with pytest.raises(api.SvsdfError) as e:
            ctx.map_clearance(*bad)
        assert "status -1" in str(e.value)
    # a path at x ~ 1.7e308 (the shape functor's squares overflow at every sample; no far-field bound holds, every column is evaluated):
    # a non-finite svsdf_query value is SVSDF_ERR_NONFINITE, finite ones are listed as for any path
    b = np.zeros((6, 3))
    b[0, 0] = b[5, 0] = 1.7e308
    T1, co1 = np.array([1.0]), b.T.reshape(-1).copy()
    ij, xy, sdf, ts = dense_values(ctx, T1, co1, occ, origin, res)
    if np.all(np.isfinite(sdf)):
        assert_same(ctx.map_clearance(T1, co1), clearance_oracle.summarise(ij, xy, sdf, ts, math.inf, len(ij)))
    else:
        with pytest.raises(api.SvsdfError) as e:
            ctx.map_clearance(T1, co1)
        assert "status -4" in str(e.value)
    ctx.close()


@pytest.fixture(scope="module")
def star_scene():
    g = np.load(os.path.join(GOLD, "map_star_pcd.npz"))
    res, ks = float(g["occupancy_resolution"]), int(g["kernel_size"])
    cmap = plan.gridmap3d_from_cloud(g["points"], res, int(g["sta_threshold"]))
    return g, cmap, dict(kernel_size=ks, traj_parlength=float(g["traj_parlength"]))


def new_ctx():
    return api.Context("star", weight_p=scenes.YAML["weight_p"], safety_hor=scenes.YAML["safety_hor"], rho=scenes.YAML["rho"])


def same_value(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same_value(a[k], b[k]) for k in a)
    if isinstance(a, np.ndarray):
        return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))
    if isinstance(a, float):
        return bits(a) == bits(b)
    return a == b


def test_certified_plans(star_scene):
    g, cmap, kw = star_scene
    ctx = new_ctx()
    p0 = plan.generate_traj(ctx, cmap, g["start"][:2], g["end"][:2], **kw)
    p1 = plan.generate_traj(ctx, cmap, g["start"][:2], g["end"][:2], certify=True, **kw)
    assert p1.keys() == p0.keys() | {"clearance"}
    for k in p0:
        if k != "seconds":
            assert same_value(p0[k], p1[k]), k
    c = p1["clearance"]
    T, co = p1["T"], np.asarray(p1["coeffs"]).reshape(-1)
    ij, xy, sdf, ts = dense_values(ctx, T, co, cmap.occ, cmap.boundary_min[:2], cmap.res)
    d = clearance_oracle.summarise(ij, xy, sdf, ts, scenes.YAML["safety_hor"], len(ij))
    assert bits(c["min_sdf"]) == bits(d["min_sdf"]) and c["collision_free"] == (d["min_sdf"] > 0)
    assert (c["n_within"], c["n_colliding"]) == (d["n_within"], d["n_colliding"]) and c["n_evaluated"] <= len(ij)
    if d["argmin"] >= 0:
        assert np.array_equal(bits(c["argmin_xy"]), bits(d["xy"][d["argmin"]])) and bits(c["t_star"]) == bits(d["tstar"][d["argmin"]])
    else:
        assert c["argmin_xy"] is None and c["t_star"] is None
    # plan_batch: every problem that went through the back end carries generate_traj(certify=True)'s clearance
    free = np.argwhere(~cmap.occ.any(axis=2))
    pick = free[np.random.default_rng(5).choice(len(free), size=(5, 2), replace=False)]
    xy2 = cmap.boundary_min[:2] + (pick + 0.5) * cmap.res
    starts, goals = np.r_[[g["start"][:2]], xy2[:, 0]], np.r_[[g["end"][:2]], xy2[:, 1]]
    stats = {}
    batch = plan.plan_batch(new_ctx(), cmap, starts, goals, certify=True, stats=stats, **kw)
    assert stats["certify_s"] > 0.0
    n = 0
    for s, e, r in zip(starts, goals, batch):
        alone = plan.generate_traj(ctx, cmap, s, e, certify=True, **kw)
        assert ("clearance" in r) == ("clearance" in alone) == ("T" in r)
        if "clearance" in r:
            assert same_value(r["clearance"], alone["clearance"])
            n += 1
    assert n >= 2
    ctx.close()
