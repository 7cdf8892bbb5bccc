"""GPU parity tests of the A* front end's collision kernels (SURVEY.md §8f rank 3; csrc/svsdf_frontend.cu) through the C ABI:
svsdf_front_init / _get_kernels (BasicShape::initShape), svsdf_front_cspace (kernelConv over the whole configuration space),
svsdf_front_check_kernel_value (checkKernelValue).  Integer / byte work: everything is compared bit for bit with the oracle.
The oracle is itself held to the reference's own node test and search by tests/test_oracle_front_ref_pin.py, and
tests/test_gpu_front_edges.py takes every entry point to the limits of its inputs (resolutions, box sizes, map shapes, yaw
counts and father yaws) against both."""
import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, batch

pytestmark = pytest.mark.gpu

ANALYTIC = ["star", "sdHorseshoe", "sdPie", "sdPie2", "sdArc", "sdTunnel", "sdCutDisk", "sdTrapezoid", "sdRhombus", "sdHeart",
            "sdRoundedX", "bigX", "sdRoundedCross", "sdOrientedVesica", "sdMoon", "sdUnevenCapsule", "Circle"]


def random_occ(X, Y, density, seed):
    rng = np.random.default_rng(seed)
    return rng.random((X, Y)) < density


def test_shape_kernels_are_bitwise_the_oracles(oracle_mod):
    for pp in ((0.0, 0.0, 0.0), (0.4, -0.2, 25.0)):
        for name in ANALYTIC:
            for ks, K, res, safeh in ((17, 18, 1.0, 0.0), (31, 36, 0.2, 0.15)):
                ctx = api.Context(name, poly_params=pp)
                ctx.front_init(ks, K, res, safeh)
                yaw, cells, byt = ctx.front_kernels()
                yaw_o, cells_o, byt_o = oracle_mod.shape_kernels(name, ks, K, res, safeh, poly_params=pp)
                assert np.array_equal(yaw, yaw_o)
                assert np.array_equal(cells, cells_o), (name, pp, ks, int((cells != cells_o).sum()))
                assert np.array_equal(byt, byt_o)
                ctx.close()


@pytest.mark.parametrize("X,Y,ks,K,density", [(50, 61, 17, 18, 0.03), (33, 32, 9, 8, 0.08), (7, 100, 5, 4, 0.1), (64, 257, 31, 36, 0.01),
                                              (40, 40, 17, 18, 0.0), (20, 31, 3, 64, 0.3)])
def test_cspace_is_bitwise_kernel_conv(oracle_mod, X, Y, ks, K, density):
    occ = random_occ(X, Y, density, X * 1000 + Y)
    res = 0.3
    ctx = api.Context("sdHorseshoe")
    ctx.front_init(ks, K, res, 0.05)
    ctx.set_map(batch.pack_map_kernel(occ, ks), X, Y, ks, (0.0, 0.0), res)
    free, ms = ctx.front_cspace(X, Y)
    want = oracle_mod.cspace("sdHorseshoe", occ, ks, K, res, 0.05, variant="byte")
    assert free.shape == want.shape and np.array_equal(free, want)
    if density == 0.0:
        assert free.all()
    # checkKernelValue on every cell / a spread of father yaws: literal device restatement vs the oracle, and vs lookups in the map above
    rng = np.random.default_rng(1)
    n = 3000
    ind = np.stack([rng.integers(0, X, n), rng.integers(0, Y, n)], axis=1)
    fy = rng.uniform(-3.14, 3.14, n)
    ok, cy = ctx.front_check_kernel_value(fy, ind)
    ok_o, cy_o = oracle_mod.check_kernel_value("sdHorseshoe", occ, fy, ind, ks, K, res, 0.05)
    assert np.array_equal(ok, ok_o) and np.array_equal(cy[ok], cy_o[ok])
    ctx.close()


def test_front_end_errors(oracle_mod):
    ctx = api.Context("unknown_shape_falls_back_to_polygon")
    with pytest.raises(api.SvsdfError):
        ctx.front_init(17, 18, 1.0, 0.0)
    ctx.close()
    ctx = api.Context("star")
    with pytest.raises(api.SvsdfError):
        ctx.front_init(16, 18, 1.0, 0.0)  # even kernel size
    ctx._front = (17, 18)
    with pytest.raises(api.SvsdfError):
        ctx.front_cspace(10, 10)  # not initialised
    ctx.front_init(17, 18, 1.0, 0.0)
    with pytest.raises(api.SvsdfError):
        ctx.front_cspace(10, 10)  # no map
    occ = random_occ(10, 10, 0.1, 0)
    ctx.set_map(batch.pack_map_kernel(occ, 9), 10, 10, 9, (0.0, 0.0), 1.0)
    with pytest.raises(api.SvsdfError):
        ctx.front_cspace(10, 10)  # map packed for another kernel size
    ctx.set_map(batch.pack_map_kernel(occ, 17), 10, 10, 17, (0.0, 0.0), 1.0)
    with pytest.raises(api.SvsdfError):
        ctx.front_check_kernel_value([0.0], [[10, 3]])  # outside the map
    ctx.close()


def test_full_size_map_properties(oracle_mod):
    """2400 x 2400 cells (60 m at 0.025 m), 18 yaw kernels of 17 x 17: the size of the batch mode's map."""
    gm = batch.make_random_map(extent=60.0, res=0.025, density=0.002, seed=5)
    X, Y = gm.shape
    ks, K, res = 17, 18, 0.025
    ctx = api.Context("star")
    ctx.front_init(ks, K, res, 0.0)
    ctx.set_map(batch.pack_map_kernel(gm.occ, ks), X, Y, ks, (0.0, 0.0), res)
    free, ms = ctx.front_cspace(X, Y)
    assert free.shape == (K, X, Y)
    _, cells, _ = ctx.front_kernels()
    centre_set = cells[:, ks // 2, ks // 2]
    assert not (free[centre_set][:, gm.occ]).any()      # an occupied cell under the kernel centre is a collision
    # a crop compared with the oracle (interior of the crop: windows do not leave it)
    x0, y0, n = 700, 1300, 120
    h = (ks - 1) // 2
    crop = gm.occ[x0 - h : x0 + n + h, y0 - h : y0 + n + h]
    want = oracle_mod.cspace("star", crop, ks, K, res, 0.0)[:, h : h + n, h : h + n]
    assert np.array_equal(free[:, x0 : x0 + n, y0 : y0 + n], want)
    # the literal per-node test agrees with look-ups in the map
    rng = np.random.default_rng(3)
    m = 100_000
    ind = np.stack([rng.integers(0, X, m), rng.integers(0, Y, m)], axis=1)
    fy = rng.uniform(-3.14, 3.14, m)
    ok, cy = ctx.front_check_kernel_value(fy, ind)
    pi = 3.1415926536
    fi = np.clip((K * ((fy + pi) / (2 * pi))).astype(int), 0, K - 1)
    order = np.stack([fi] + [v for d in range(1, 6) for v in ((fi - d) % K, (fi + d) % K)], axis=1)  # breadth-first ring
    hits = free[order, ind[:, :1], ind[:, 1:]]
    assert np.array_equal(ok, hits.any(axis=1))
    first = order[np.arange(m), hits.argmax(axis=1)]
    assert np.array_equal(cy[ok], (2 * pi * first / K - pi)[ok])
    ctx.close()


@pytest.mark.parametrize("shape,pp", [("star", (0.0, 0.0, 0.0)), ("sdHorseshoe", (0.0, 0.0, 0.0)), ("sdTunnel", (0.3, -0.2, 20.0))])
def test_expand_nodes_is_bitwise_the_oracles(oracle_mod, shape, pp):
    """AstarPathSearcher::process neighbour loop (kernel test + sub-swept-volume test) for a batch of nodes."""
    X, Y, ks, K, res = 70, 55, 17, 18, 1.0
    occ = random_occ(X, Y, 0.012, 99)
    origin = (-12.5, 3.25)
    rng = np.random.default_rng(4)
    n = 400
    ij = np.stack([rng.integers(0, X, n), rng.integers(0, Y, n)], axis=1)
    ij[:6] = [[0, 0], [X - 1, Y - 1], [0, Y - 1], [X - 1, 0], [X // 2, 0], [0, Y // 2]]  # map corners and edges
    fy = rng.uniform(-3.14, 3.14, n)
    ctx = api.Context(shape, poly_params=pp)
    ctx.front_init(ks, K, res, 0.0)
    ctx.set_map(batch.pack_map_kernel(occ, ks), X, Y, ks, origin, res)
    ok, cy, parts = ctx.front_expand(ij, fy)
    ok_o, cy_o, parts_o = oracle_mod.expand_nodes(shape, occ, ij, fy, origin=origin, map_res=res, kernel_size=ks, kernel_count=K, safeh=0.0,
                                                  poly_params=pp)
    assert np.array_equal(parts, parts_o), int((parts != parts_o).sum())
    assert np.array_equal(ok, ok_o) and np.array_equal(cy, cy_o)
    assert 0.05 < ok.mean() < 0.99  # the scene exercises both outcomes
    assert len(np.unique(parts)) >= 4
    ctx.close()


def test_batch_astar_equals_the_oracles_search(oracle_mod):
    """svsdf_front_astar: n searches in lock-step on the GPU node test vs the oracle's literal AstarPathSearch per problem."""
    rng = np.random.default_rng(33)
    X, Y, ks, K, res = 60, 52, 17, 18, 1.0
    occ = rng.random((X, Y)) < 0.005
    origin = (2.0, -9.5)
    n = 64
    st = np.c_[rng.uniform(origin[0], origin[0] + X, n), rng.uniform(origin[1], origin[1] + Y, n)]
    go = np.c_[rng.uniform(origin[0], origin[0] + X, n), rng.uniform(origin[1], origin[1] + Y, n)]
    st[3] = [origin[0] - 2.0, origin[1] + 1.0]  # outside the map
    ctx = api.Context("star")
    ctx.front_init(ks, K, res, 0.0)
    ctx.set_map(batch.pack_map_kernel(occ, ks), X, Y, ks, origin, res)
    paths, ex, rounds = ctx.front_astar(st, go)
    paths_o, ex_o = oracle_mod.astar("star", occ, st, go, origin=origin, map_res=res, kernel_size=ks, kernel_count=K)
    assert np.array_equal(ex, ex_o)
    found = 0
    for p, po in zip(paths, paths_o):
        assert (p is None) == (po is None)
        if p is not None:
            assert np.array_equal(p, po)
            found += 1
    assert found >= n // 2 and paths[3] is None
    assert rounds == ex.max() + 0 or rounds >= ex.max()  # lock-step: as many rounds as the longest search needs (+ its goal pop)
    ctx.close()
