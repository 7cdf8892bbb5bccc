"""GPU (-m gpu): the pose-sampled obstacle penalty's kernel (k_pose, strict build) against the REFERENCE'S OWN grad_cost_p
(tests/golden/ref_pin_pose.npz, tests/golden/make_pose_golden.py) at every recorded pose: every analytic shape and the Polygon, with
and without poly_params, on the star map and a five-layer map, with poses outside the map, boxes clipped at every face, yaws
selecting one, all or no layers, voxels exactly at |p_rel| = half and the four smoothed-L1 regimes.  A pose p is fed to the kernel as
a piece whose only non-zero coefficients are c_0 = p: with integralIntervs = 1 both of its samples sit at p.  Also: the batch pool
(svsdf_optimize_batch) carries each context's setting, and plan_batch equals generate_traj per problem with the term on."""
import os
import sys

import numpy as np
import pytest

from implicit_svsdf_planner_b200 import api, plan, scenes
from oracle import k3_points

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_gpu_lockstep as L  # noqa: E402
import test_gpu_optimize_device as OD  # noqa: E402
import test_gpu_dynamics as DY  # noqa: E402  (the star scene and its free start / goal pairs)
import test_oracle_pose_ref_pin as PIN  # noqa: E402  (the golden's cases)

pytestmark = pytest.mark.gpu
KS = 3
PARAMS = OD.PARAMS


def set_map(ctx, gm):
    X, Y, Z = gm.size
    ctx.set_map3d(k3_points.generate_map_kernel(gm, KS), X, Y, Z, KS, gm.boundary_min, gm.res)


def kernel_records(ctx, poses, half):
    """k_pose's records at the poses (svsdf_pose_penalty_eval, one piece per pose, integralIntervs = 1): both samples of each piece."""
    out0, out1 = [], []
    for s in range(0, len(poses), 64):
        P = poses[s:s + 64]
        N = len(P)
        b = np.zeros((6 * N, 3))
        b[0::6] = P
        _, _, _, rec = ctx.pose_penalty(np.ones(N), np.ascontiguousarray(b.T).reshape(-1),
                                        dict(weight=60.0, integralIntervs=1, half=half), samples=True)
        out0.append(rec[0::2])
        out1.append(rec[1::2])
    return np.concatenate(out0), np.concatenate(out1)


@pytest.mark.parametrize("mi", [0, 1])
@pytest.mark.parametrize("pi", [0, 1])
def test_strict_kernel_is_the_reference(mi, pi):
    gm, half = PIN.MAPS[mi]
    pp = PIN.G["case_pp"][pi]
    checked = 0
    for k, cmi, shape, cpp, poses, rec in PIN.CASES:
        if cmi != mi or tuple(cpp) != tuple(pp):
            continue
        ctx = api.Context(shape, poly_params=tuple(pp), safety_hor=float(PIN.G["safety_hor"]), strict_fp=True)
        set_map(ctx, gm)
        r0, r1 = kernel_records(ctx, poses, half)
        ctx.close()
        assert np.array_equal(L.bits(r0), L.bits(rec)), (shape, pp, np.argwhere(L.bits(r0) != L.bits(rec))[:5])
        assert np.array_equal(L.bits(r1), L.bits(rec)), (shape, pp)
        checked += 1
    assert checked == 18


def test_optimize_batch_pool_carries_each_contexts_setting():
    gm = k3_points.GridMap3D(np.array([-10.0, -16.0, -2.0]), np.array([200.0, 20.0, 2.0]), 1.0,
                             np.random.default_rng(3).random((210, 36, 4)) < 0.02)
    probs = [OD.problem(8, 40, 81), OD.problem(8, 60, 82), OD.problem(8, 0, 83)]
    on, off = L.ctx_for("star"), L.ctx_for("star")
    for c in (on, off):
        set_map(c, gm)
    on.set_pose_penalty()
    ref_on = [L.run_single(on, p, PARAMS) for p in probs]
    ref_off = [L.run_single(off, p, PARAMS) for p in probs]
    assert any(a["final_cost"] != b["final_cost"] for a, b in zip(ref_on, ref_off))
    for ctx, ref in ((on, ref_on), (off, ref_off)):
        _, X, _, status, _ = api.optimize_batch([ctx], [dict(init_s=p["init_s"], final_s=p["final_s"], x0=p["x0"], points=p["points"])
                                                        for p in probs], 8, PARAMS)
        for k, r in enumerate(ref):
            assert np.array_equal(L.bits(X[k]), L.bits(r["x"])) and status[k] == r["status"], k
    on.close()
    off.close()


def ctx_new(pose):
    ctx = api.Context("star", weight_p=scenes.YAML["weight_p"], safety_hor=scenes.YAML["safety_hor"], rho=scenes.YAML["rho"])
    ctx.set_pose_penalty(pose)
    return ctx


@pytest.mark.parametrize("n", [12, 256])
def test_plan_batch_is_generate_traj_with_the_pose_penalty(n):
    """n < 256 runs the host lock-step back end, n >= 256 the device back end; each problem equals generate_traj's bits."""
    g, cmap, kw = DY.star_scene()
    st, go = DY.free_pairs(cmap, n, 5 + n)
    st[0], go[0] = g["start"][:2], g["end"][:2]
    pose = api.yaml_pose_penalty(scenes.YAML)
    ctx = ctx_new(pose)
    got = plan.plan_batch(ctx, cmap, st, go, **kw)
    checked = 0
    for q in range(n) if n < 256 else list(range(0, n, 37)) + [n - 1]:
        r = plan.generate_traj(ctx_new(pose), cmap, st[q], go[q], **kw)
        b = got[q]
        assert b["ok"] == r["ok"], q
        if "T" not in r:
            continue
        for key in ("x", "T", "coeffs"):
            assert np.array_equal(L.bits(b[key]), L.bits(r[key])), (q, key)
        assert (b["iterations"], b["evaluations"], b["status"]) == (r["iterations"], r["evaluations"], r["status"]), q
        checked += 1
    assert checked >= 3
    ctx.close()
