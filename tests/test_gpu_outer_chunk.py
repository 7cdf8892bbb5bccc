"""GPU tests of the batched k_outer's chunked descent pass (run with -m gpu on an H100): a CTA seeds up to KernelArgs::outer_chunk
batches of every warp, drains them in ONE descent_engine2 pass over one queue and then finishes the batches in their own order.

The chunk changes which group of lanes solves a point and when, never what is computed, and the per-warp accumulation keeps its
batch order.  So under the test hook SVSDF_FORCE_OUTER_CHUNK = 1, 2, 3, 4 (read when a context is created) every output of
svsdf_query (sdf, t*, gradient, rounds) and of svsdf_cost_grad / svsdf_cost_grad_multi (cost, gradT, gradC, interior count) must be
BYTEWISE the one of chunk 1, and chunk 1 must give the recorded bits of the reference's own code on the edge scenes
(tests/golden/ref_pin_outer_edges.npz).  Strict and FMA build.
"""
import os
import sys

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, scenes

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
sys.path.insert(0, GOLD)
import make_outer_edges_golden as mko  # noqa: E402

CHUNKS = (1, 2, 3, 4)
HOOKS = ("SVSDF_FORCE_OUTER_CHUNK", "SVSDF_FORCE_BATCHED", "SVSDF_FORCE_GRID_OUTER", "SVSDF_FORCE_GSIP_WIDE", "SVSDF_FORCE_GRID_GSIP",
         "SVSDF_FORCE_POSE_WINDOWS")


def _set(monkeypatch, chunk=None, batched=None, grid=None):
    for var, val in zip(HOOKS, (chunk, batched, grid, None, None, None)):
        if val is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, str(val))


def pts3(p):
    p = np.atleast_2d(np.asarray(p, dtype=np.float64))
    return np.c_[p[:, :2], np.zeros(len(p))]


def _bytes(x):
    return np.ascontiguousarray(x).tobytes()


def _same(got, ref, what):
    assert len(got) == len(ref), what
    for i, (a, b) in enumerate(zip(got, ref)):
        assert _bytes(a) == _bytes(b), (what, "output", i)


def _evaluate(monkeypatch, chunk, batched, grid, shape, T, co, pts, scale=None, **kw):
    """Query and cost of one problem on a context created under the hooks: (sdf, t*, gradient, rounds, cost, gradT, gradC)."""
    _set(monkeypatch, chunk, batched, grid)
    if shape == "star_obj_mesh":
        g = np.load(os.path.join(GOLD, "fwn_ref.npz"))
        ctx = api.Context("star", mesh=(g["star_V"], g["star_F"]), **kw)
    else:
        ctx = api.Context(shape, **kw)
    _set(monkeypatch)
    try:
        if scale is not None:
            ctx.set_scale(**scale)
        q = ctx.query(T, co, pts3(pts))
        ctx.set_points(pts3(pts))
        c, gT, gC = ctx.cost_grad(T, co)
        return (*q, np.float64(c), gT, gC)
    finally:
        ctx.close()


def _every_chunk_equals_chunk_1(monkeypatch, what, batched, grid, shape, T, co, pts, **kw):
    ref = _evaluate(monkeypatch, 1, batched, grid, shape, T, co, pts, **kw)
    for chunk in CHUNKS[1:]:
        _same(_evaluate(monkeypatch, chunk, batched, grid, shape, T, co, pts, **kw), ref, (what, chunk))
    return ref


SC = {}


def scene(name):
    if name not in SC:
        SC[name] = {"config2": lambda: scenes.make_scene("star", 8, 200_000), "scene2k": lambda: scenes.make_scene("star", 8, 2000),
                    "small_inside": lambda: scenes.make_scene("star", 8, 400, clearance=2.35)}[name]()
    return SC[name]


@pytest.mark.parametrize("strict_fp", [True, False], ids=["strict", "fma"])
def test_config2_production_grid(monkeypatch, strict_fp):
    """Star, 8 pieces, 200 000 points, no schedule hook: two batches per warp, so the production chunk is 2 (one pass per CTA); the
    unforced context gives the same bytes as every forced chunk."""
    sc = scene("config2")
    kw = dict(weight_p=sc.weight_p, safety_hor=sc.safety_hor, strict_fp=strict_fp)
    ref = _every_chunk_equals_chunk_1(monkeypatch, "config2", None, None, "star", sc.T, sc.coeffs_colmajor(), sc.points, **kw)
    _same(_evaluate(monkeypatch, None, None, None, "star", sc.T, sc.coeffs_colmajor(), sc.points, **kw), ref, "config2 unforced")
    assert (ref[3] > 0).any() and ref[4] > 0  # interior points and a penalty


@pytest.mark.parametrize("grid", [1, 3, 37])
def test_rounds_that_are_not_a_multiple_of_the_chunk(monkeypatch, grid):
    """2000 points, batched on 1, 3 and 37 CTAs: 8, 3 and 1 batches per warp, so the last pass of a CTA holds fewer batches than the
    chunk (3 = 2 + 1, 8 = 3 + 3 + 2) or the chunk exceeds the rounds altogether."""
    sc = scene("scene2k")
    _every_chunk_equals_chunk_1(monkeypatch, ("scene2k", grid), 1, grid, "star", sc.T, sc.coeffs_colmajor(), sc.points,
                                weight_p=sc.weight_p, safety_hor=sc.safety_hor)


@pytest.mark.parametrize("P,grid", [(5, 1), (37, 1), (300, 1), (700, 2)])
def test_batches_with_fewer_than_32_points(monkeypatch, P, grid):
    """Batches of 0-1, 4-5 and 18-19 points (holes in every chunk of the queue), and 21-22 points over 2 rounds on 2 CTAs."""
    sc = scene("small_inside") if P <= 400 else scene("scene2k")
    _every_chunk_equals_chunk_1(monkeypatch, ("ragged", P), 1, grid, "star", sc.T, sc.coeffs_colmajor(), sc.points[:P],
                                weight_p=sc.weight_p, safety_hor=sc.safety_hor)


@pytest.mark.parametrize("P", [383, 384])
def test_batched_threshold_pair(monkeypatch, P):
    """P = 128 g - 1 (sparse: the chunk is not read) and P = 128 g (batched) on g = 3 CTAs, the runtime's own rule."""
    sc = scene("scene2k")
    _every_chunk_equals_chunk_1(monkeypatch, ("threshold", P), None, 3, "star", sc.T, sc.coeffs_colmajor(), sc.points[:P],
                                weight_p=sc.weight_p, safety_hor=sc.safety_hor)


def test_largest_trajectory_where_one_round_clips_the_chunk(monkeypatch):
    """N = 64, D = 299.84 s: about 176 KB of shared memory with one work area and one CTA per SM.  20 000 points are one batch per
    warp on the production grid (the chunk is clipped to 1); on a forced grid of 8 CTAs they are 10, with up to 32 KB of work area."""
    shape, T, co, _ = mko.scene("long64")
    pts = mko.long64_points(20_000, 70 + 20_000)
    ref = _every_chunk_equals_chunk_1(monkeypatch, "long64", None, None, shape, T, co, pts)
    _same(_every_chunk_equals_chunk_1(monkeypatch, "long64 grid 8", 1, 8, shape, T, co, pts)[:4], ref[:4], "long64 grids")


@pytest.mark.parametrize("case", ["scaled", "star_obj_mesh"])
def test_scaled_and_mesh_kernels(monkeypatch, case):
    """k_outer_scaled (deformable robot) and the triangle-mesh functor, batched on one CTA: 2 rounds."""
    sc = scene("small_inside")
    shape = "star" if case == "scaled" else "star_obj_mesh"
    scale = api.EXAMPLE_SCALE if case == "scaled" else None
    ref = _every_chunk_equals_chunk_1(monkeypatch, case, 1, 1, shape, sc.T, sc.coeffs_colmajor(), sc.points, scale=scale,
                                      weight_p=sc.weight_p, safety_hor=sc.safety_hor)
    assert ref[4] > 0


@pytest.mark.parametrize("scale", [None, api.EXAMPLE_SCALE], ids=["rigid", "scaled"])
def test_mixed_multi_batch(monkeypatch, scale):
    """svsdf_cost_grad_multi over problems of 1, 8 and 64 pieces with 1 to 2000 points, every one batched on its own virtual grid of
    up to 2 CTAs (1 to 4 rounds): the launch's chunk is the one of its largest shared-memory class, and every record is bytewise the
    one of chunk 1 and of the problem's single call."""
    _, T1, co1, p1 = mko.scene("tiny_k1")
    sc, sk = scene("small_inside"), scene("scene2k")
    _, T64, co64, p64 = mko.scene("long64")
    probs = [(T1, co1, pts3(p1[:1])), (sc.T, sc.coeffs_colmajor(), pts3(sc.points[:300])), (T64, co64, pts3(p64[:1000])),
             (sk.T, sk.coeffs_colmajor(), pts3(sk.points))]
    res = {}
    for chunk in CHUNKS:
        _set(monkeypatch, chunk, 1, 2)
        ctx = api.Context("star", weight_p=sc.weight_p, safety_hor=sc.safety_hor)
        _set(monkeypatch)
        if scale is not None:
            ctx.set_scale(**scale)
        res[chunk] = [(np.float64(c), gT, gC, np.int64(ni)) for c, gT, gC, ni in ctx.cost_grad_multi(probs)]
        if chunk == 1:
            for (T, co, pts), rec in zip(probs, res[1]):
                ctx.set_points(pts)
                c, gT, gC = ctx.cost_grad(T, co)
                _same((np.float64(c), gT, gC), rec[:3], ("multi against single", len(T)))
        ctx.close()
    for chunk in CHUNKS[1:]:
        for k, (a, b) in enumerate(zip(res[chunk], res[1])):
            _same(a, b, ("multi", chunk, k))
    assert sum(r[3] for r in res[1]) > 0


@pytest.mark.parametrize("chunk", CHUNKS)
def test_edge_scenes_are_bitwise_the_reference_code(monkeypatch, chunk):
    """Every edge scene of the outer solve, batched on one CTA (up to 8 rounds), against the recorded outputs of the reference's own
    code ("portable" variant): full query and outer-only query."""
    g = np.load(os.path.join(GOLD, "ref_pin_outer_edges.npz"))
    for key in mko.SCENES:
        shape, T, co, pts = str(g[f"{key}_shape"]), g[f"{key}_T"], g[f"{key}_coeffs"], g[f"{key}_points"]
        _set(monkeypatch, chunk, 1, 1)
        ctx = api.Context(shape, strict_fp=True)
        _set(monkeypatch)
        for outer_only, pre in ((False, ""), (True, "o")):
            got = ctx.query(T, co, pts, outer_only=outer_only)[:3]
            for a, n in zip(got, ("sdf", "tstar", "grad")):
                ref = g[f"{key}_{pre}{n}_portable"]
                assert _bytes(a + 0.0) == _bytes(ref.reshape(a.shape) + 0.0), (key, chunk, pre + n)  # +-0 equal
        ctx.close()
