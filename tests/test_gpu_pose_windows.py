"""GPU tests of the pose windows of choiceTInit layers 2 and 3 (k_pose_table, svsdf_types.h:PoseRec): the poses of every layer-2
window (one per layer-1 winner kb, kb = -1 included) and of every layer-3 window (one per kb and layer-2 sample m2, m2 = none
included), which thread_choice_t_init (batched schedule) and solve_outer (sparse schedule, k_gsip's ring samples) read instead of
evaluating the trajectory.

Per point sdf, t* and gradient must be BIT FOR BIT those of the same context type without windows, under the test hook
SVSDF_FORCE_POSE_WINDOWS (read when a context is created): 0 = none, 1 = layer 2, 2 = layers 2 and 3, unset = the rule of
pose_windows() (the layer-3 windows only when they hold at most two records per layer-3 sample of the P points).  The scenes are the outer
solve's edge scenes (tests/golden/make_outer_edges_golden.py); a host replay of the scan loops checks that they reach the windows
this is about: clamped at 0 and at D, kb = -1, layer 2 finding no improvement, one piece and 64 pieces.
"""
import os
import sys

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_outer_edges_golden as mko  # noqa: E402

HOOKS = ("SVSDF_FORCE_POSE_WINDOWS", "SVSDF_FORCE_BATCHED", "SVSDF_FORCE_GRID_OUTER", "SVSDF_FORCE_GSIP_WIDE", "SVSDF_FORCE_GRID_GSIP")
SCHEDULES = {"sparse": ("0", None), "batched_grid3": ("1", "3")}
KWINLEN = 21


def _set(monkeypatch, windows=None, batched=None, grid=None):
    for var, val in zip(HOOKS, (windows, batched, grid, None, None)):
        if val is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, val)


def _query(shape, T, co, pts, outer_only=False):
    ctx = api.Context(shape, strict_fp=True)
    try:
        return ctx.query(T, co, pts, outer_only=outer_only)
    finally:
        ctx.close()


def _assert_same(got, ref, what):
    for a, b, n in zip(got, ref, ("sdf", "t*", "gradient", "rounds")):
        a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
        if a.dtype == np.float64:
            a, b = a + 0.0, b + 0.0  # +-0 equal
            same = a.view(np.int64) == b.view(np.int64)
        else:
            same = a == b
        if not same.all():
            bad = np.flatnonzero(~same.reshape(len(a), -1).all(axis=1))
            raise AssertionError(f"{what}: {n} differs at {bad.size} points, first {bad[:5]}")


def replay(orc, p, D, lat):
    """choiceTInit's layers 1-3 on the host for one point: (kb, m2, layer-2 window, layer-3 window), each window as
    (start clamped at 0, end clamped at D, sample count)."""
    vals = [orc.sdf_at(p, t) for t in lat]
    min_dis, kb = 1e9, -1
    for k, d in enumerate(vals):
        if d < min_dis:
            min_dis, kb = d, k
    seed = lat[kb] if kb >= 0 else 0.0
    wins, m2 = [], None
    for layer in (2, 3):
        ts = mko.layer_times(seed, D, layer)
        dt = 0.15 * 0.1 if layer == 2 else 0.15 * 0.1 * 0.1
        wins.append((seed - 10 * dt < 0.0, seed + 10 * dt > D, len(ts)))
        for m, t in enumerate(ts):
            d = orc.sdf_at(p, t)
            if d < min_dis:
                seed, min_dis = t, d
                if layer == 2:
                    m2 = m
    return kb, m2, wins[0], wins[1]


def test_every_window_fits_its_record_row():
    """Every layer-2 window (kb = -1 .. K1 - 1) and every layer-3 window (every kb and m2) of the 1-piece, 2-piece and 64-piece
    scenes holds at most 21 samples: the fixed row of kWinLen records the kernels index by sample number."""
    for name in ("tiny_k1", "tiny_n2", "long64", "broken"):
        _, T, _, _ = mko.scene(name)
        D = 0.0
        for d in T:
            D += d
        lat = mko.lattice(D)
        for seed2 in [0.0] + lat:
            w2 = mko.layer_times(seed2, D, 2)
            assert 1 <= len(w2) <= KWINLEN, (name, seed2, len(w2))
            for seed3 in [seed2] + w2:
                assert 1 <= len(mko.layer_times(seed3, D, 3)) <= KWINLEN, (name, seed2, seed3)


def test_edge_scenes_reach_the_windows_under_test(oracle_mod):
    """The host replay of the scan loops on the small edge scenes: layer-2 and layer-3 windows clamped at 0 and at D, points with
    nothing below 1e9 (kb = -1), and layer 2 both finding and not finding a lower sample (m2 = none)."""
    seen = dict(kb_none=0, m2_none=0, m2_some=0, w2_at0=0, w2_atD=0, w3_at0=0, w3_atD=0)
    for name in ("tiny_k1", "tiny_k21", "tiny_n2", "parked", "far", "broken"):
        shape, T, co, pts = mko.scene(name)
        orc = oracle_mod.Oracle(shape, threads=1)
        orc.set_traj(np.asarray(T, float), co)
        D = orc.duration()
        lat = mko.lattice(D)
        for p in pts[:: max(1, len(pts) // 60)]:
            kb, m2, w2, w3 = replay(orc, p, D, lat)
            seen["kb_none"] += kb < 0
            seen["m2_none"] += m2 is None
            seen["m2_some"] += m2 is not None
            seen["w2_at0"] += w2[0]
            seen["w2_atD"] += w2[1]
            seen["w3_at0"] += w3[0]
            seen["w3_atD"] += w3[1]
    print(seen)
    assert min(seen.values()) >= 1, seen


@pytest.mark.parametrize("schedule", list(SCHEDULES))
def test_windows_on_and_off_give_the_same_bits(monkeypatch, schedule):
    """Every edge scene, full query (outer solve and interior branch) and outer-only query: no windows, layer 2, layers 2 and 3
    and the production rule, bit for bit."""
    for name in mko.SCENES:
        shape, T, co, pts = mko.scene(name)
        _set(monkeypatch, "0", *SCHEDULES[schedule])
        ref, ref_o = _query(shape, T, co, pts), _query(shape, T, co, pts, outer_only=True)
        for windows in ("1", "2", None):
            _set(monkeypatch, windows, *SCHEDULES[schedule])
            _assert_same(_query(shape, T, co, pts), ref, (name, schedule, windows))
            _assert_same(_query(shape, T, co, pts, outer_only=True), ref_o, (name, schedule, windows, "outer_only"))


@pytest.mark.parametrize("P", [5_000, 200_000], ids=["rule_layer2_only", "rule_layers2and3"])
def test_long_trajectory_on_both_sides_of_the_layer3_rule(monkeypatch, P):
    """N = 64, D = 299.84 s (K1 = 1999: 924 000 layer-3 records, built from 22 000 points on): 5 000 points stay below the
    rule's threshold (layer 2 only), 200 000 are above it.  The production choice, the layer-3 windows forced on and the windows forced off agree bit for bit,
    per point and in the cost and gradient."""
    shape, T, co, _ = mko.scene("long64")
    pts = mko.long64_points(P, 90 + P)
    out = {}
    for windows in ("0", "2", None):
        _set(monkeypatch, windows)
        ctx = api.Context(shape, strict_fp=True)
        q = ctx.query(T, co, pts)
        ctx.set_points(pts)
        out[windows] = (q, ctx.cost_grad(T, co))
        ctx.close()
    for windows in ("2", None):
        _assert_same(out[windows][0], out["0"][0], ("long64", P, windows))
        for a, b in zip(out[windows][1], out["0"][1]):
            assert np.array_equal(np.asarray(a) + 0.0, np.asarray(b) + 0.0), ("long64", P, windows)
