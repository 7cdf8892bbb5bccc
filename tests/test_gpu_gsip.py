"""GPU tests of the interior (GSIP) branch of getTrueSDFofSweptVolume<true> (run with -m gpu on an H100): k_compact (ordered
compaction of the interior flags), both instantiations of k_gsip (8 warps per CTA, or 22 warps = one warp per ring sample,
picked when the previous cost evaluation had at most one interior point per SM) and the interior part of k_finalize.

The strict build computes every interior point with the oracle's operations in the oracle's order: the same ring samples,
the same outer solves, the same arg-max, the same world -> body rotation in the penalty.  So sdf, t*, gradient and round count
are compared BIT FOR BIT for every point, in both k_gsip variants and with k_gsip's grid forced to one CTA (which walks every
slot) and to three (a ragged split) — SVSDF_FORCE_GSIP_WIDE / SVSDF_FORCE_GRID_GSIP, read when a context is created.

The scene builders assert, with the oracle on the CPU, the branches each scene exists for, so that a later edit to a scene
cannot silently drop coverage: the velocity fallback scanning forward (t* < 0.1, |v| < 0.01), scanning backward
(t* > D - 0.1), or not scanning at all (a slow t* in the middle of the trajectory), the 9-round cap of the ring search, an
outer sdf of exactly 0.0, and interior points at both ends of a 40 009-point set.
"""
import json
import os
import sys

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, scenes

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
sys.path.insert(0, GOLD)
import make_gsip_edges_golden as mkg  # noqa: E402  (inputs of the edge scenes, shared with the reference fixture)

ALL_SHAPES = ["star", "sdHorseshoe", "sdPie", "sdPie2", "sdArc", "sdTunnel", "sdCutDisk", "sdTrapezoid", "sdRhombus",
              "sdHeart", "sdRoundedX", "bigX", "sdRoundedCross", "sdOrientedVesica", "sdMoon", "sdUnevenCapsule",
              "Circle", "unknown_mesh_shape"]
PRE = ((0.0, 0.0, 0.0), (0.4, -0.25, 33.0))
WIDE = {"8warp": "0", "22warp": "1"}
P_DENSE = 40_009
STALE_P = 37  # points 37..47 of the dense scene are interior: the last flag word of a 37-point set holds their stale flags
# An H100 SM holds at most 2048 threads = 8 CTAs of k_gsip's 256: more interior points than this walks several slots per CTA
# on the default grid whatever the occupancy
MAX_GSIP_CTAS = 132 * 8


def nrel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def gT_err(gT, gT_ref, gC_ref):
    """gradT error on the scale of its terms (see test_gpu_parity.gT_err)."""
    return np.linalg.norm(np.asarray(gT) - gT_ref) / (np.linalg.norm(gT_ref) + 1e-3 * np.linalg.norm(gC_ref))


def bits_differ(a, b):
    """Number of elements whose bit patterns differ, -0.0 and +0.0 counted as equal (test_gpu_ref_pin.bits_differ)."""
    a = np.ascontiguousarray(a, dtype=np.float64).ravel() + 0.0
    b = np.ascontiguousarray(b, dtype=np.float64).ravel() + 0.0
    assert a.shape == b.shape
    return int((a.view(np.int64) != b.view(np.int64)).sum())


def star_traj():
    init_s, final_s, q, T = scenes.make_trajectory("star", 8)
    b = scenes.minco_dense(init_s, final_s, q, T)
    return T, b


def scatter_points(n, seed):
    """n points within +-3 m of the star trajectory: most of them inside its swept volume."""
    T, b = star_traj()
    path = scenes.eval_traj_xy(b, T, np.linspace(0.0, float(T.sum()), 2000))[:, :2]
    rng = np.random.default_rng(seed)
    xy = path[rng.integers(0, 2000, n)] + rng.uniform(-3.0, 3.0, (n, 2))
    return np.c_[xy, np.zeros(n)]


class Scene:
    """Inputs of one scene + the oracle's per-point results and the branch classification of its interior points."""

    def __init__(self, O, name, T, co, pts, shape="star", **kw):
        self.name, self.T, self.co, self.pts, self.shape, self.kw = name, np.asarray(T, float), co, pts, shape, kw
        orc = O.Oracle(shape, threads=O.num_procs(), **kw)
        orc.set_traj(self.T, co)
        self.ref = orc.query(pts)
        so, to, _ = orc.query_outer(pts)
        D = float(self.T.sum())
        self.inside = ~(so > 0)
        assert np.array_equal(self.inside, self.ref[3] > 0)
        slow = np.zeros(len(pts), dtype=bool)
        for k in np.flatnonzero(self.inside):  # k_gsip: `if (sqrt(vx * vx + vy * vy + vw * vw) < 0.01)` at the outer t*
            v = orc.traj_vel(to[k])
            slow[k] = np.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]) < 0.01
        self.forward = slow & (to < 0.1)
        self.backward = slow & ~(to < 0.1) & (to > D - 0.1)
        self.slow_mid = slow & ~self.forward & ~self.backward
        self.zero = so == 0.0
        self.nine = self.ref[3] == 9

    def context(self, **kw):
        return api.Context(self.shape, strict_fp=kw.pop("strict_fp", True), **self.kw, **kw)

    def coverage(self):
        return dict(P=len(self.pts), inside=int(self.inside.sum()), forward=int(self.forward.sum()),
                    backward=int(self.backward.sum()), slow_mid=int(self.slow_mid.sum()), zero=int(self.zero.sum()),
                    nine_rounds=int(self.nine.sum()))


def build_edge_scene(O, name):
    if name == "small_inside":
        sc = scenes.make_scene("star", 8, 400, clearance=2.35)
        s = Scene(O, name, sc.T, sc.coeffs_colmajor(), np.c_[sc.points[:, :2], np.zeros(sc.P)])
        assert s.inside.sum() >= 20 and s.forward.sum() >= 1 and s.backward.sum() >= 1, s.coverage()
        return s
    if name == "dense":
        return build_dense_scene(O)
    shape, T, co, pts = mkg.scene(name)
    s = Scene(O, name, T, co, pts, shape=shape)
    c = s.coverage()
    if name == "endpoints":
        assert c["forward"] >= 10 and c["backward"] >= 10, c
    elif name == "midstop":
        assert c["slow_mid"] >= 3 and c["nine_rounds"] >= 1, c
    elif name == "circle_static":
        assert c["inside"] == c["P"] and c["zero"] >= 4 and c["forward"] == c["P"], c
    elif name == "circle_spin":
        assert c["inside"] == c["P"] and c["slow_mid"] + c["forward"] + c["backward"] == 0, c
    return s


def build_dense_scene(O):
    """P = 40 009 (more than one 16-byte flag word per k_compact thread; P % 16 = 9): a map scene plus points scattered around
    the path, interior points moved to indices 0, 37..47 and P - 1."""
    sc = scenes.make_scene("star", 8, P_DENSE - 1809)
    rng = np.random.default_rng(31)
    pts = np.r_[np.c_[sc.points[:, :2], np.zeros(sc.P)], scatter_points(1809, 32)]
    pts = pts[rng.permutation(P_DENSE)]
    orc = O.Oracle("star", threads=O.num_procs())
    orc.set_traj(sc.T, sc.coeffs_colmajor())
    inside = ~(orc.query_outer(pts)[0] > 0)
    targets = [0, *range(STALE_P, 48), P_DENSE - 1]
    spare = [k for k in np.flatnonzero(inside) if k not in targets]
    for t in targets:
        if not inside[t]:
            k = spare.pop()
            pts[[t, k]] = pts[[k, t]]
    s = Scene(O, "dense", sc.T, sc.coeffs_colmajor(), pts)
    assert len(s.pts) == P_DENSE and s.inside[targets].all(), s.coverage()
    assert s.inside.sum() > MAX_GSIP_CTAS, s.coverage()
    return s


EDGE_SCENES = ("small_inside", "endpoints", "midstop", "circle_static", "circle_spin", "dense")


@pytest.fixture(scope="module")
def edge(oracle_mod):
    out = {name: build_edge_scene(oracle_mod, name) for name in EDGE_SCENES}
    for s in out.values():
        print(s.name, s.coverage())
    return out


def _set_hooks(monkeypatch, wide=None, grid=None):
    for var, val in (("SVSDF_FORCE_GSIP_WIDE", wide), ("SVSDF_FORCE_GRID_GSIP", grid)):
        if val is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, val)


def _assert_query_bitwise(got, ref, what):
    names = ("sdf", "t*", "gradient", "rounds")
    for a, b, n in zip(got, ref, names):
        if not np.array_equal(a, b):
            bad = np.flatnonzero((a != b).reshape(len(a), -1).any(axis=1))
            raise AssertionError(f"{what}: {n} differs at {bad.size} points, first {bad[:5]}: {a[bad[:3]]} vs {b[bad[:3]]}")


# ---------------------------------------------------------------------------------------------------------------------
# per point, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid", [None, "1", "3"], ids=["grid_default", "grid_1", "grid_3"])
@pytest.mark.parametrize("variant", list(WIDE))
def test_every_point_of_the_edge_scenes_is_bitwise_the_oracle(edge, monkeypatch, variant, grid):
    _set_hooks(monkeypatch, WIDE[variant], grid)
    for s in edge.values():
        ctx = s.context()
        got = ctx.query(s.T, s.co, s.pts)
        _assert_query_bitwise(got, s.ref, (s.name, variant, grid))
        ctx.close()


@pytest.mark.parametrize("variant", list(WIDE))
def test_edge_scenes_are_bitwise_the_reference_code(monkeypatch, variant):
    """The edge scenes against the reference's own code (tests/golden/ref_pin_gsip_edges.npz, "portable" variant): the kernels
    reproduce it per point, outer solve and interior branch alike."""
    _set_hooks(monkeypatch, WIDE[variant])
    g = np.load(os.path.join(GOLD, "ref_pin_gsip_edges.npz"))
    for key in mkg.SCENES:
        shape, T, co, pts = str(g[f"{key}_shape"]), g[f"{key}_T"], g[f"{key}_coeffs"], g[f"{key}_points"]
        ctx = api.Context(shape, strict_fp=True)
        sdf, tstar, grad, rounds = ctx.query(T, co, pts)
        assert bits_differ(sdf, g[f"{key}_sdf_portable"]) == 0, key
        assert bits_differ(tstar, g[f"{key}_tstar_portable"]) == 0, key
        assert bits_differ(grad, g[f"{key}_grad_portable"]) == 0, key
        assert np.array_equal(rounds > 0, ~(g[f"{key}_osdf_portable"] > 0)), key
        so, to, go, _ = ctx.query(T, co, pts, outer_only=True)
        assert bits_differ(so, g[f"{key}_osdf_portable"]) + bits_differ(to, g[f"{key}_otstar_portable"]) \
            + bits_differ(go, g[f"{key}_ograd_portable"]) == 0, key
        ctx.close()


def _shape_case(name):
    """(Context / Oracle keyword arguments, points) of one functor of the every-shape test."""
    if name == "star_obj_mesh":  # the oracle's mesh functor is slow: 44 points, about 40 of them interior, some at the ends
        g = np.load(os.path.join(GOLD, "fwn_ref.npz"))
        return dict(mesh=(g["star_V"], g["star_F"])), np.r_[scatter_points(24, 42), mkg.scene("endpoints")[3][::6]]
    if name == "star_outline_polygon":  # BASELINE config 4: the outline of shapes/star.obj through the Polygon functor
        xy = np.array(json.load(open(os.path.join(GOLD, "obj_outlines.json")))["star"]["outline_xy"])
        return dict(polygon=xy[np.argsort(np.arctan2(xy[:, 1], xy[:, 0]))].reshape(-1)), scatter_points(1500, 41)
    return {}, scatter_points(1500, 41)


@pytest.mark.parametrize("name", ALL_SHAPES + ["star_obj_mesh", "star_outline_polygon"])
def test_every_shape_interior_points_are_bitwise(oracle_mod, monkeypatch, name):
    """Every functor (16 registry shapes, Circle, the Polygon fallback, the reference's star.obj mesh, config 4's star outline)
    with and without a body-frame pre-transform, both k_gsip variants: interior points included, every output bitwise."""
    kw, pts = _shape_case(name)
    T, b = star_traj()
    co = np.ascontiguousarray(b.T).reshape(-1)
    scans = 0
    for pp in PRE:
        s = Scene(oracle_mod, name, T, co, pts, shape=name, poly_params=pp, **kw)
        c = s.coverage()
        assert c["inside"] >= 20, (name, pp, c)
        scans += c["forward"] + c["backward"]
        for variant, flag in WIDE.items():
            _set_hooks(monkeypatch, flag)
            ctx = s.context()
            _assert_query_bitwise(ctx.query(T, co, pts), s.ref, (name, pp, variant))
            ctx.close()
    assert scans >= 1, name  # the velocity fallback scan is reached for every functor


# ---------------------------------------------------------------------------------------------------------------------
# the interior contribution path: k_gsip -> gsip_contrib / gsip_piece -> k_finalize
# ---------------------------------------------------------------------------------------------------------------------
def _pick_interior(s, n):
    """Up to n interior points of a scene, the special ones (scans, slow t*, outer sdf 0, 9 rounds) first."""
    order = []
    for m in (s.forward, s.backward, s.slow_mid, s.zero & s.inside, s.nine, s.inside):
        order += [int(k) for k in np.flatnonzero(m) if k not in order]
    return order[:n]


def test_single_interior_point_cost_is_bitwise_the_oracle(edge, oracle_mod, monkeypatch):
    """With a single point there is no summation order: k_outer's partials are exact zeros and k_finalize adds zeros to the
    one contribution, so cost, gradC and gradT equal the oracle's bits (+-0 equal).  Each point is evaluated twice on one
    context: the first evaluation runs the 8-warp k_gsip (no previous count), the second the 22-warp one (one interior point
    <= SMs).  Interior points take the world -> body rotation of the gradient (`sdf < 0`) and add gdT to gradT(j), j < piece."""
    _set_hooks(monkeypatch)
    n_checked = 0
    for s in edge.values():
        orc = oracle_mod.Oracle(s.shape, threads=1, **s.kw)
        ctx = s.context()
        for k in _pick_interior(s, 12):
            p = s.pts[k : k + 1]
            orc.set_points(p)
            c0, gT0, gC0, _, n_in = orc.cost_grad(s.T, s.co)
            assert n_in == 1 and c0 > 0, (s.name, k)
            ctx.set_points(p)
            for call in ("8warp", "22warp"):
                c1, gT1, gC1 = ctx.cost_grad(s.T, s.co)
                assert c1 == c0 and np.array_equal(gC1, gC0) and np.array_equal(gT1, gT0), (s.name, k, call, c1, c0)
            n_checked += 1
        ctx.close()
    assert n_checked >= 60


def test_adaptive_variant_switch_and_inside_count(edge, oracle_mod, monkeypatch):
    """cost_grad twice on one set: the second evaluation switches to the 22-warp k_gsip when the first saw <= SMs interior
    points (small_inside) and stays on the 8-warp one otherwise (dense); both give the same bits.  The inside count the
    device reports is the oracle's, and the sums agree with the oracle's to summation order."""
    _set_hooks(monkeypatch)
    for name in ("small_inside", "dense"):
        s = edge[name]
        n_in = int(s.inside.sum())
        assert (0 < n_in <= 132) if name == "small_inside" else (n_in > 132), (name, n_in)
        ctx = s.context()
        ctx.set_points(s.pts)
        c1, gT1, gC1 = ctx.cost_grad(s.T, s.co)
        c2, gT2, gC2 = ctx.cost_grad(s.T, s.co)
        assert c1 == c2 and np.array_equal(gT1, gT2) and np.array_equal(gC1, gC2), name
        _, out = ctx.cost_grad_device(s.T, s.co)
        N = len(s.T)
        assert int(out[1 + 19 * N]) == n_in, (name, out[1 + 19 * N], n_in)
        assert out[0] == c1 and np.array_equal(out[1 : 1 + 18 * N], gC1), name
        orc = oracle_mod.Oracle(s.shape, threads=oracle_mod.num_procs(), **s.kw)
        orc.set_points(s.pts)
        c0, gT0, gC0, _, inside = orc.cost_grad(s.T, s.co)
        assert inside == n_in
        assert abs(c1 - c0) <= 1e-12 * abs(c0), (name, c1, c0)
        assert nrel(gC1, gC0) <= 1e-12 and gT_err(gT1, gT0, gC0) <= 1e-12, (name, nrel(gC1, gC0), gT_err(gT1, gT0, gC0))
        ctx.close()


def test_stale_flags_of_a_larger_set_do_not_leak(edge, monkeypatch):
    """The flag scratch only grows: after the 40 009-point set, a 37-point set finds the dense set's interior flags 37..47 in
    its last 16-byte flag word.  k_compact must mask them (tail beyond P); query and cost equal a fresh context's bits."""
    _set_hooks(monkeypatch)
    d = edge["dense"]
    small = d.pts[:STALE_P]
    assert d.inside[STALE_P:48].all() and d.inside[:STALE_P].any()
    fresh = d.context()
    want_q = fresh.query(d.T, d.co, small)
    fresh.set_points(small)
    want_c = fresh.cost_grad(d.T, d.co)
    fresh.close()
    _assert_query_bitwise(want_q, tuple(a[:STALE_P] for a in d.ref), "fresh context")
    ctx = d.context()
    ctx.query(d.T, d.co, d.pts)
    _assert_query_bitwise(ctx.query(d.T, d.co, small), want_q, "after the dense query")
    ctx.set_points(d.pts)
    ctx.cost_grad(d.T, d.co)
    ctx.set_points(small)
    c, gT, gC = ctx.cost_grad(d.T, d.co)
    assert c == want_c[0] and np.array_equal(gT, want_c[1]) and np.array_equal(gC, want_c[2]), (c, want_c[0])
    ctx.close()


def test_fma_build_with_the_wide_variant_stays_within_the_reference_noise_floor(edge, oracle_mod, monkeypatch):
    """strict_fp = 0 with the 22-warp k_gsip forced: inside the same noise floor as the 8-warp path
    (test_gpu_parity.test_cost_grad_fma_build_stays_within_the_reference_noise_floor)."""
    _set_hooks(monkeypatch, "1")
    s = edge["small_inside"]
    ctx = s.context(strict_fp=False)
    ctx.set_points(s.pts)
    c1, gT1, gC1 = ctx.cost_grad(s.T, s.co)
    ctx.close()
    for variant in ("default", "fma"):
        o = oracle_mod.Oracle("star", threads=oracle_mod.num_procs(), variant=variant)
        o.set_points(s.pts)
        c0, gT0, gC0, _, _ = o.cost_grad(s.T, s.co)
        assert abs(c1 - c0) <= 1e-9 * abs(c0), (variant, c1, c0)
        assert nrel(gC1, gC0) <= 1e-4, (variant, nrel(gC1, gC0))
