"""GPU (-m gpu): svsdf_front_astar_device — whole A* searches on the device, one launch for n searches (csrc/svsdf_frontend.cu
k_astar_search around csrc/host/astar_flat.hpp).  Everything is compared bit for bit: path x, y and yaw, lengths, expansion counts
and status, against the oracle's literal AstarPathSearch (with an expansion budget and branch counters through
tests/astar_oracle_ext.py) and the lock-step svsdf_front_astar."""
import os

import numpy as np
import pytest

import astar_oracle_ext
from implicit_svsdf_planner_b200 import api, batch, plan, scenes

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
KS, K, RES = 17, 18, 1.0


def context(shape, occ, origin, pp=(0.0, 0.0, 0.0)):
    X, Y = occ.shape
    ctx = api.Context(shape, poly_params=pp)
    ctx.front_init(KS, K, RES, 0.0)
    ctx.set_map(batch.pack_map_kernel(occ, KS), X, Y, KS, origin, RES)
    return ctx


def in_map(p, occ, origin):
    X, Y = occ.shape
    return not (p[0] < origin[0] or p[1] < origin[1] or p[0] > origin[0] + X * RES or p[1] > origin[1] + Y * RES)


def oracle_expect(shape, occ, st, go, origin, pp=(0.0, 0.0, 0.0), max_path=1024, max_expansions=None):
    """(paths, expansions, status) the device call must return, from the oracle's search (run with room for any path)."""
    X, Y = occ.shape
    full, ex = astar_oracle_ext.astar(shape, occ, st, go, origin=origin, map_res=RES, kernel_size=KS, kernel_count=K, max_path=X * Y + 1,
                                poly_params=pp, max_expansions=max_expansions)
    paths, status = [], np.zeros(len(full), dtype=np.int32)
    for q, p in enumerate(full):
        if not (in_map(st[q], occ, origin) and in_map(go[q], occ, origin)):
            status[q] = 0
        elif p is not None:
            status[q] = 1 if len(p) <= max_path else 4
        else:
            status[q] = 3 if (max_expansions is not None and ex[q] == max_expansions) else 2
        paths.append(p if (p is not None and len(p) <= max_path) else None)
    return paths, ex, status


def assert_same(got, want):
    paths, ex, status = got[:3]
    paths_w, ex_w, status_w = want
    assert np.array_equal(ex, ex_w), np.nonzero(ex != ex_w)
    assert np.array_equal(status, status_w), np.nonzero(status != status_w)
    for q, (p, pw) in enumerate(zip(paths, paths_w)):
        assert (p is None) == (pw is None), q
        if p is not None:
            assert p.shape == pw.shape and np.array_equal(p, pw), q


def parity_scene():
    """The scene of test_batch_astar_equals_the_oracles_search: 60 x 52 cells, 64 searches, search 3 starts outside the map."""
    rng = np.random.default_rng(33)
    X, Y = 60, 52
    occ = rng.random((X, Y)) < 0.005
    origin = (2.0, -9.5)
    n = 64
    st = np.c_[rng.uniform(origin[0], origin[0] + X, n), rng.uniform(origin[1], origin[1] + Y, n)]
    go = np.c_[rng.uniform(origin[0], origin[0] + X, n), rng.uniform(origin[1], origin[1] + Y, n)]
    st[3] = [origin[0] - 2.0, origin[1] + 1.0]
    return occ, origin, st, go


PARITY = [("star", (0.0, 0.0, 0.0)), ("sdHorseshoe", (0.0, 0.0, 0.0)), ("sdTunnel", (0.3, -0.2, 20.0))]


@pytest.mark.parametrize("shape,pp", PARITY)
def test_device_search_equals_the_oracle_and_the_lockstep_search(shape, pp):
    occ, origin, st, go = parity_scene()
    # the scene reaches the search's quirky branches (oracle counters, per search): closed nodes re-opened, open nodes improved
    # without re-keying, pops decided by insertion order among equal f
    _, _, cnt = astar_oracle_ext.astar(shape, occ, st, go, origin=origin, map_res=RES, kernel_size=KS, kernel_count=K, poly_params=pp, counts=True)
    assert (cnt.sum(axis=0) >= 1).all(), cnt.sum(axis=0)
    ctx = context(shape, occ, origin, pp)
    got = ctx.front_astar_device(st, go)
    want = oracle_expect(shape, occ, st, go, origin, pp)
    assert_same(got, want)
    assert got[2][3] == 0 and (got[2] == 1).sum() >= len(st) // 2
    paths_l, ex_l, _ = ctx.front_astar(st, go)
    assert np.array_equal(ex_l, got[1])
    assert all((a is None) == (b is None) and (a is None or np.array_equal(a, b)) for a, b in zip(paths_l, got[0]))
    assert got[3] > 0.0
    ctx.close()


def edge_scene():
    """The parity scene's map with a goal cell walled in by a ring of obstacles around cell (44, 12) and one occupied cell (10, 40)."""
    occ, origin, _, _ = parity_scene()
    occ = occ.copy()
    occ[40:49, 8:17] = True
    occ[41:48, 9:16] = False
    occ[10, 40] = True
    return occ, origin


def cell_centre(origin, i, j):
    return [origin[0] + (i + 0.5) * RES, origin[1] + (j + 0.5) * RES]


def test_edge_cases_equal_the_oracle():
    occ, origin = edge_scene()
    X, Y = occ.shape
    c = lambda i, j: cell_centre(origin, i, j)
    top = [origin[0] + X * RES, origin[1] + Y * RES]  # exactly on the upper boundary: inside by isInMap, index clamps to the last cell
    cases = [
        (c(12, 12), [origin[0] + 12.9, origin[1] + 12.1]),  # start and goal in the same cell
        (c(15, 30), c(44, 12)),                             # goal enclosed by obstacles
        (c(15, 30), c(10, 40)),                             # goal cell occupied
        ([top[0], origin[1] + 26.3], c(20, 20)),            # start on the upper x boundary
        (c(28, 30), [origin[0] + 30.0, top[1]]),            # goal on the upper y boundary
        (top, c(30, 30)),                                   # start on the upper corner
        (c(8, 8), c(50, 44)),                               # a long search
    ]
    st = np.array([a for a, _ in cases])
    go = np.array([b for _, b in cases])
    ctx = context("star", occ, origin)
    got = ctx.front_astar_device(st, go)
    want = oracle_expect("star", occ, st, go, origin)
    assert_same(got, want)
    paths, ex, status, _ = got
    assert len(paths[0]) == 1 and ex[0] == 0 and status[0] == 1
    assert status[1] == 2 and ex[1] > 0 and status[2] == 2
    assert (status[3:] == 1).all()
    assert np.array_equal(paths[3][0, :2], cell_centre(origin, X - 1, 26)) and np.array_equal(paths[4][-1, :2], cell_centre(origin, 30, Y - 1))
    assert np.array_equal(paths[5][0, :2], cell_centre(origin, X - 1, Y - 1))
    L = 6
    long_len, long_ex = len(paths[L]), int(ex[L])
    # max_path one shorter than the path: status 4, length 0
    got = ctx.front_astar_device(st[L:], go[L:], max_path=long_len - 1)
    assert got[0][0] is None and got[1][0] == long_ex and got[2][0] == 4
    assert_same(got, oracle_expect("star", occ, st[L:], go[L:], origin, max_path=long_len - 1))
    # a budget below the oracle's count: status 3 after exactly k expansions, like the oracle's max_expansions
    for k in (1, long_ex // 2, long_ex - 1):
        got = ctx.front_astar_device(st[L:], go[L:], max_expansions=k)
        assert got[0][0] is None and got[1][0] == k and got[2][0] == 3
        assert_same(got, oracle_expect("star", occ, st[L:], go[L:], origin, max_expansions=k))
    # the exact count the search needs: the goal pop comes before the budget test
    got = ctx.front_astar_device(st[L:], go[L:], max_expansions=long_ex)
    assert got[2][0] == 1 and got[1][0] == long_ex and np.array_equal(got[0][0], paths[L])
    # the enclosed goal with a budget above its count still ends on an empty open list
    got = ctx.front_astar_device(st[1:2], go[1:2], max_expansions=int(ex[1]) + 1)
    assert got[2][0] == 2 and got[1][0] == ex[1]
    ctx.close()


def mixed_set():
    occ, origin, st, go = parity_scene()
    st2, go2 = st.copy(), go.copy()
    st2[::5] = go2[::5] + 0.1  # short searches (same or neighbouring cell) between the long ones
    return occ, origin, np.r_[st, st2], np.r_[go, go2]


def test_work_queue_grid_does_not_change_results(monkeypatch):
    occ, origin, st, go = mixed_set()
    outs = []
    for g in (None, "1", "3"):
        if g is None:
            monkeypatch.delenv("SVSDF_FORCE_GRID_ASTAR", raising=False)
        else:
            monkeypatch.setenv("SVSDF_FORCE_GRID_ASTAR", g)  # read once by svsdf_create
        ctx = context("star", occ, origin)
        outs.append(ctx.front_astar_device(st, go))
        ctx.close()
    monkeypatch.delenv("SVSDF_FORCE_GRID_ASTAR", raising=False)
    for o in outs[1:]:
        assert_same(o, outs[0][:3])
    assert_same(outs[0], oracle_expect("star", occ, st, go, origin))


def test_context_reuse_across_map_sizes_matches_fresh_contexts():
    rng = np.random.default_rng(21)
    big = rng.random((60, 60)) < 0.01
    small = rng.random((30, 25)) < 0.01
    n = 96
    sb = rng.uniform(0.0, 60.0, size=(n, 2)), rng.uniform(0.0, 60.0, size=(n, 2))
    ss = np.c_[rng.uniform(0, 30, n), rng.uniform(0, 25, n)], np.c_[rng.uniform(0, 30, n), rng.uniform(0, 25, n)]
    fresh = []
    for occ, (st, go) in ((big, sb), (small, ss)):
        ctx = context("sdHorseshoe", occ, (0.0, 0.0))
        fresh.append(ctx.front_astar_device(st, go))
        ctx.close()
    ctx = context("sdHorseshoe", big, (0.0, 0.0))
    for occ, (st, go), want in ((big, sb, fresh[0]), (small, ss, fresh[1]), (big, sb, fresh[0])):
        X, Y = occ.shape
        ctx.set_map(batch.pack_map_kernel(occ, KS), X, Y, KS, (0.0, 0.0), RES)
        assert_same(ctx.front_astar_device(st, go), want[:3])
    ctx.close()


def test_1024_searches_equal_the_lockstep_search():
    rng = np.random.default_rng(7)
    occ = rng.random((60, 60)) < 0.005
    st, go = rng.uniform(1.0, 59.0, size=(1024, 2)), rng.uniform(1.0, 59.0, size=(1024, 2))
    ctx = context("star", occ, (0.0, 0.0))
    launches0 = ctx.kernel_launches()
    paths, ex, status, ms = ctx.front_astar_device(st, go)
    assert ctx.kernel_launches() == launches0 + 1  # one launch for all 1024 searches
    paths_l, ex_l, _ = ctx.front_astar(st, go)
    assert np.array_equal(ex, ex_l)
    for p, pl, s in zip(paths, paths_l, status):
        assert (p is None) == (pl is None) and (p is None or np.array_equal(p, pl))
        assert s == (1 if p is not None else 2)
    ctx.close()


def test_star_scene_search_equals_the_lockstep_search():
    g = np.load(os.path.join(HERE, "golden", "map_star_pcd.npz"))
    res, ks = float(g["occupancy_resolution"]), int(g["kernel_size"])
    cmap = plan.gridmap3d_from_cloud(g["points"], res, int(g["sta_threshold"]))
    X, Y, Z = cmap.occ.shape
    ctx = api.Context("star", weight_p=scenes.YAML["weight_p"], safety_hor=scenes.YAML["safety_hor"], rho=scenes.YAML["rho"])
    ctx.set_map3d(plan.pack_map_kernel3d(cmap.occ, ks), X, Y, Z, ks, cmap.boundary_min, res)
    ctx.front_init(ks, 18, res, 0.0)
    st, go = g["start"][:2].reshape(1, 2), g["end"][:2].reshape(1, 2)
    paths_l, ex_l, _ = ctx.front_astar(st, go, 4096)
    paths, ex, status, _ = ctx.front_astar_device(st, go, 4096)
    assert status[0] == 1 and ex[0] == ex_l[0] and np.array_equal(paths[0], paths_l[0])
    ctx.close()


def test_errors_raise_without_a_device_fault():
    occ, origin = edge_scene()
    X, Y = occ.shape
    st, go = np.array([cell_centre(origin, 2, 2)]), np.array([cell_centre(origin, 5, 9)])
    ctx = api.Context("star")
    with pytest.raises(api.SvsdfError, match="front_init"):
        ctx.front_astar_device(st, go)  # no front_init
    ctx.front_init(KS, K, RES, 0.0)
    with pytest.raises(api.SvsdfError, match="map not set"):
        ctx.front_astar_device(st, go)
    ctx.set_map(batch.pack_map_kernel(occ, 9), X, Y, 9, origin, RES)
    with pytest.raises(api.SvsdfError, match="another kernel_size"):
        ctx.front_astar_device(st, go)
    ctx.set_map(batch.pack_map_kernel(occ, KS), X, Y, KS, origin, RES)
    with pytest.raises(api.SvsdfError):
        ctx.front_astar_device(st, go, max_path=0)
    with pytest.raises(api.SvsdfError):
        ctx.front_astar_device(st, go, max_expansions=0)
    paths, ex, status, ms = ctx.front_astar_device(np.zeros((0, 2)), np.zeros((0, 2)))
    assert paths == [] and ex.shape == (0,) and status.shape == (0,)
    paths, ex, status, _ = ctx.front_astar_device(st, go)  # the context still works
    assert status[0] == 1
    ctx.close()
    poly = api.Context("unknown_shape_falls_back_to_polygon")
    with pytest.raises(api.SvsdfError):
        poly.front_init(KS, K, RES, 0.0)
    poly.set_map(batch.pack_map_kernel(occ, KS), X, Y, KS, origin, RES)
    with pytest.raises(api.SvsdfError, match="front_init"):
        poly.front_astar_device(st, go)
    poly.close()
