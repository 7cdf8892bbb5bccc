"""CPU: the oracle's A* (oracle/frontend_oracle.hpp astar_search) with a per-search expansion budget and the per-search branch
counters the device-search scene builders rely on (tests/astar_oracle_ext.py), checked against oracle_py.astar."""
import numpy as np

import astar_oracle_ext


def scene():
    rng = np.random.default_rng(33)
    X, Y = 60, 52
    occ = rng.random((X, Y)) < 0.005
    origin = (2.0, -9.5)
    n = 24
    st = np.c_[rng.uniform(origin[0], origin[0] + X, n), rng.uniform(origin[1], origin[1] + Y, n)]
    go = np.c_[rng.uniform(origin[0], origin[0] + X, n), rng.uniform(origin[1], origin[1] + Y, n)]
    return occ, origin, st, go


def same(a, b):
    return all((p is None) == (q is None) and (p is None or np.array_equal(p, q)) for p, q in zip(a, b))


def test_oracle_astar_max_expansions_passthrough(oracle_mod):
    occ, origin, st, go = scene()
    paths, ex = oracle_mod.astar("star", occ, st, go, origin=origin)
    # no budget, and the instrumented copy run beside it, give oracle_py.astar's searches
    paths2, ex2, cnt = astar_oracle_ext.astar("star", occ, st, go, origin=origin, counts=True)
    assert np.array_equal(ex, ex2) and same(paths, paths2) and cnt.shape == (len(st), 3)
    q = int(np.argmax(np.where([p is not None for p in paths], ex, -1)))
    k = int(ex[q])
    assert paths[q] is not None and k > 2
    for budget in (1, k // 2, k - 1):  # the budget test comes after the goal test: below the count there is no path
        pb, eb, _ = astar_oracle_ext.astar("star", occ, st[q:q + 1], go[q:q + 1], origin=origin, max_expansions=budget, counts=True)
        assert pb[0] is None and eb[0] == budget
    pb, eb = astar_oracle_ext.astar("star", occ, st[q:q + 1], go[q:q + 1], origin=origin, max_expansions=k)  # exactly enough
    assert eb[0] == k and np.array_equal(pb[0], paths[q])


def test_oracle_astar_counts_the_quirky_branches():
    occ, origin, st, go = scene()
    _, ex, cnt = astar_oracle_ext.astar("star", occ, st, go, origin=origin, counts=True)
    assert (cnt >= 0).all() and (cnt.sum(axis=0) >= 1).all(), cnt.sum(axis=0)
    assert (cnt[ex == 0] == 0).all()  # a search that expands nothing re-opens and improves nothing
