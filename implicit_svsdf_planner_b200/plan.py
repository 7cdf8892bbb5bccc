"""One plan from point cloud to optimised trajectory: the chain PlannerManager::generatePath / generateTraj drives in the reference
(src/plan_manager/src/plan_manager.cpp:96-227), on this build's entry points.

  point cloud -> occupancy grid                 PCSmapManager::rcvGlobalMapHandler      map_manager/src/PCSmap_manager.cpp:113-190
  grid -> byte-packed maps                      generateMapKernel / generateMapKernel2D  map_manager/include/map_manager/PCSmap_manager.h:39-108
  A* over (x, y, yaw) with the shape kernels    AstarPathSearcher::AstarPathSearch       -> svsdf_front_astar (GPU node tests)
  path -> waypoints, boxes -> query points      generateTraj                             plan_manager.cpp:131-175 -> svsdf_extract_points3d (GPU)
  warm start                                    OriTraj::getOriTraj                      -> svsdf_mid_get_ori_traj (host)
  SVSDF back end                                TrajOptimizer::optimize_traj_lmbm        -> svsdf_optimize (GPU cost + gradient, host solver)

Host-side glue only (numpy); every arithmetic step is behind the C ABI.  The map construction and the waypoint rule are checked against
oracle/k3_points.py by tests/test_oracle_k3.py, the chain itself by tests/test_gpu_plan.py on the reference's own star scene."""
from __future__ import annotations

import concurrent.futures as cf
import dataclasses
import math
import time
from typing import Optional

import numpy as np

from . import api, scenes


@dataclasses.dataclass
class CloudMap:
    occ: np.ndarray            # [X, Y, Z] bool
    boundary_min: np.ndarray   # boundary_xyzmin
    boundary_max: np.ndarray   # boundary_xyzmax
    res: float


def gridmap3d_from_cloud(points_f32, res: float, sta_threshold: int = 1) -> CloudMap:
    """rcvGlobalMapHandler: boundary = min / max of the cloud (pcl::PointXYZ floats widened to double), size = ceil(extent / res)
    (Gridmap3D.cpp:25-41), a voxel is occupied when at least sta_threshold points fall into it; index = floor((p - min) / res) clamped to
    the last cell (Gridmap3D.cpp:137-174; every cloud point is inside the boundary by construction)."""
    pts = np.asarray(points_f32, dtype=np.float32).astype(np.float64).reshape(-1, 3)
    lo, hi = pts.min(axis=0), pts.max(axis=0)
    size = np.maximum(np.ceil((hi - lo) / res).astype(np.int64), 0)
    cnt = np.zeros(tuple(int(s) for s in size), dtype=np.int64)
    if cnt.size:
        idx = np.floor((pts - lo) / res).astype(np.int64)
        idx = np.minimum(np.maximum(idx, 0), size - 1)
        np.add.at(cnt, (idx[:, 0], idx[:, 1], idx[:, 2]), 1)
    return CloudMap(occ=cnt >= sta_threshold, boundary_min=lo, boundary_max=hi, res=float(res))


def pack_map_kernel3d(occ: np.ndarray, kernel_size: int) -> np.ndarray:
    """generateMapKernel (PCSmap_manager.h:39-78): [(X + 2h)][(Y + 2h)][ceil((Z + 2h) / 8)] bytes, z bits MSB first."""
    h = (kernel_size - 1) // 2
    X, Y, Z = occ.shape
    bits = np.zeros((X + 2 * h, Y + 2 * h, 8 * ((Z + 2 * h + 7) // 8)), dtype=np.uint8)
    bits[h:h + X, h:h + Y, h:h + Z] = occ
    return np.packbits(bits, axis=2)  # MSB first, as or_mask = {0x80, ..., 0x01}


def waypoints_of_path(path: np.ndarray, traj_parlength: float, res: float):
    """plan_manager.cpp:131-158: index_gap = ceil(traj_parlength / res), shrunk by 1.5 until the path has more cells than one gap; every
    index_gap-th node of the front-end path (ends excluded) becomes a waypoint.  Returns (indices, waypoints)."""
    path = np.asarray(path, dtype=np.float64)
    n = path.shape[0]
    t = float(traj_parlength)
    gap = int(math.ceil(t / res))
    while gap >= n - 1:
        t /= 1.5
        gap = int(math.ceil(t / res))
    idx = np.arange(gap, n - 1, gap)
    return idx, path[idx]


def rot_z(yaw: float) -> np.ndarray:
    c, s = math.cos(yaw), math.sin(yaw)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def generate_traj(ctx: "api.Context", cmap: CloudMap, start_xy, goal_xy, kernel_size: int = scenes.YAML["kernel_size"], kernel_yaw_num: int = 18,
                  front_end_safeh: float = 0.0, traj_parlength: float = 3.0, inittime: float = scenes.YAML["inittime"],
                  mid_cfg: Optional["api.MidConfig"] = None, lbfgs_params=None, max_path: int = 4096, certify: bool = False) -> dict:
    """generatePath + generateTraj for one start / goal on the map `cmap` (the context's shape is the robot).  certify=True adds
    `clearance` (see certificate) to a result that reached the back end."""
    X, Y, Z = cmap.occ.shape
    res = cmap.res
    ctx.set_map3d(pack_map_kernel3d(cmap.occ, kernel_size), X, Y, Z, kernel_size, cmap.boundary_min, res)
    ctx.front_init(kernel_size, kernel_yaw_num, res, front_end_safeh)
    paths, expansions, rounds = ctx.front_astar(np.asarray(start_xy, dtype=np.float64).reshape(1, 2), np.asarray(goal_xy, dtype=np.float64).reshape(1, 2), max_path)
    path = paths[0]
    if path is None or len(path) < 3:
        return dict(ok=False, reason="front end found no path", expansions=int(expansions[0]))
    idx, wps = waypoints_of_path(path, traj_parlength, res)
    N = len(wps) + 1
    half = kernel_size * res / 3.0                      # bdx / 3 (plan_manager.cpp:57-59, 165)
    n_points = ctx.extract_points3d(wps, [half, half, half])  # the waypoint (x, y, yaw) is the box centre, as in the reference
    init_s, final_s = np.zeros((3, 3)), np.zeros((3, 3))
    init_s[:, 0], final_s[:, 0] = path[0], path[-1]     # plan_manager.cpp:143-147
    rots = np.stack([rot_z(p[2]) for p in wps])
    rc_mid, opt_x, T_mid, co_mid, cost_mid, it_mid = api.mid_get_ori_traj(init_s, final_s, wps.T, np.full(N, inittime), rots, mid_cfg)
    if rc_mid < 0:
        return dict(ok=False, reason=f"mid end failed ({rc_mid})", N=N, n_points=int(n_points))
    params = lbfgs_params or api.default_lbfgs_params(mem_size=16, past=3, delta=1e-6, g_epsilon=0.0, max_iterations=0, min_step=1e-32)
    f0, _ = ctx_evaluate(ctx, init_s, final_s, N, opt_x)
    rc, x, T, b, st = ctx.optimize(init_s, final_s, opt_x, N, params)  # the query points are the context's resident set (extract_points3d)
    out = dict(ok=rc >= 0, status=int(rc), N=N, n_points=int(n_points), path=path, waypoints=wps, expansions=int(expansions[0]), astar_rounds=int(rounds),
               mid=dict(status=int(rc_mid), cost=float(cost_mid), iterations=int(it_mid), T=T_mid), cost_at_warm_start=float(f0),
               final_cost=float(st["final_cost"]), iterations=int(st["iterations"]), evaluations=int(st["evaluations"]), T=T, coeffs=b, x=x,
               seconds=float(st["seconds"]))
    if certify:
        out["clearance"] = certificate(ctx, T, b)
    return out


def certificate(ctx: "api.Context", T, coeffs) -> dict:
    """The trajectory checked against every occupied cell of the context's map (svsdf_map_clearance, the reference's getMinSVSDF) with
    d_max = the context's safety_hor: the least swept-volume SDF value over the cells within the penalty's horizon, where it is reached,
    and collision_free = min_sdf > 0.  `ok` says only that the solver returned status >= 0; this says whether the robot misses the map."""
    c = ctx.map_clearance(T, np.asarray(coeffs).reshape(-1), ctx.safety_hor)
    k = c.argmin
    return dict(min_sdf=c.min_sdf, argmin_xy=c.xy[k].copy() if k >= 0 else None, t_star=float(c.tstar[k]) if k >= 0 else None,
                n_colliding=c.n_colliding, n_within=c.n_within, n_evaluated=c.n_evaluated, collision_free=bool(c.min_sdf > 0.0))


def ctx_evaluate(ctx, init_s, final_s, N, x):
    ctx.set_boundary(init_s, final_s, N)
    return ctx.evaluate(x)


# status of svsdf_front_astar_device -> why a plan_batch problem has no path
_ASTAR_REASON = {0: "start or goal outside the map", 2: "front end found no path", 3: "front end reached max_expansions",
                 4: "path longer than max_path", -1: "front end internal guard"}


def plan_batch(ctx: "api.Context", cmap: CloudMap, starts, goals, kernel_size: int = scenes.YAML["kernel_size"], kernel_yaw_num: int = 18,
               front_end_safeh: float = 0.0, traj_parlength: float = 3.0, inittime: float = scenes.YAML["inittime"],
               mid_cfg: Optional["api.MidConfig"] = None, lbfgs_params=None, max_path: int = 4096, max_in_flight: int = 0,
               workers: Optional[int] = None, stats: Optional[dict] = None, back_end: bool = True, certify: bool = False) -> list:
    """generate_traj for n start / goal pairs on one map: one device A* launch for all searches (svsdf_front_astar_device), per problem the
    waypoints, the query points (extract_points3d, on the context) and the warm start (mid_get_ori_traj, on a thread pool: the mid end is
    host code and ctypes releases the GIL), then ONE lock-step back end (svsdf_optimize_lockstep) for every problem whose mid end succeeded.
    Returns one dict per problem with generate_traj's keys (except astar_rounds) and its bits, plus the query points (`points`);
    a failed problem has ok=False and the reason (an exception of one problem's extraction or mid end fails that problem only).
    stats (optional dict) receives the wall seconds of each stage, the back end's rounds and its kernel launches.  back_end=False stops
    before the back end: the problems that would enter it are returned with its inputs (init_s, final_s, x0, points) instead.
    certify=True adds generate_traj's `clearance` to every problem that went through the back end (one svsdf_map_clearance per problem,
    after the back end; stats then also holds its wall seconds, certify_s)."""
    st = np.asarray(starts, dtype=np.float64).reshape(-1, 2)
    go = np.asarray(goals, dtype=np.float64).reshape(-1, 2)
    n = st.shape[0]
    X, Y, Z = cmap.occ.shape
    res = cmap.res
    ctx.set_map3d(pack_map_kernel3d(cmap.occ, kernel_size), X, Y, Z, kernel_size, cmap.boundary_min, res)
    ctx.front_init(kernel_size, kernel_yaw_num, res, front_end_safeh)
    out: list = [None] * n
    if n == 0:
        return out
    t0 = time.perf_counter()
    paths, expansions, status, _ = ctx.front_astar_device(st, go, max_path)
    t1 = time.perf_counter()
    half = kernel_size * res / 3.0  # bdx / 3 (plan_manager.cpp:57-59, 165)
    todo = []
    for q in range(n):
        path = paths[q]
        if status[q] != 1 or path is None or len(path) < 3:
            out[q] = dict(ok=False, reason=_ASTAR_REASON.get(int(status[q]), "front end found no path"), expansions=int(expansions[q]),
                          astar_status=int(status[q]))
            continue
        idx, wps = waypoints_of_path(path, traj_parlength, res)
        try:
            n_points = ctx.extract_points3d(wps, [half, half, half])
            pts = ctx.get_points()
        except api.SvsdfError as e:
            out[q] = dict(ok=False, reason=f"query points failed ({e})", N=len(wps) + 1, expansions=int(expansions[q]))
            continue
        init_s, final_s = np.zeros((3, 3)), np.zeros((3, 3))
        init_s[:, 0], final_s[:, 0] = path[0], path[-1]  # plan_manager.cpp:143-147
        todo.append(dict(q=q, path=path, wps=wps, N=len(wps) + 1, n_points=int(n_points), points=pts, init_s=init_s,
                         final_s=final_s))

    def mid(p):
        N = p["N"]
        rots = np.stack([rot_z(w[2]) for w in p["wps"]])
        try:
            return api.mid_get_ori_traj(p["init_s"], p["final_s"], p["wps"].T, np.full(N, inittime), rots, mid_cfg)
        except api.SvsdfError as e:  # generate_traj lets this propagate; here it fails the one problem
            return e

    t2 = time.perf_counter()
    with cf.ThreadPoolExecutor(max_workers=workers) as ex:
        mids = list(ex.map(mid, todo))
    t3 = time.perf_counter()
    back = []
    for p, m in zip(todo, mids):
        q = p["q"]
        if isinstance(m, Exception):
            out[q] = dict(ok=False, reason=f"mid end failed ({m})", N=p["N"], n_points=p["n_points"])
            continue
        rc_mid, opt_x, T_mid, co_mid, cost_mid, it_mid = m
        if rc_mid < 0:
            out[q] = dict(ok=False, reason=f"mid end failed ({rc_mid})", N=p["N"], n_points=p["n_points"])
            continue
        p["mid"] = dict(status=int(rc_mid), cost=float(cost_mid), iterations=int(it_mid), T=T_mid)
        p["x0"] = opt_x
        back.append(p)
    if not back_end:
        for p in back:
            out[p["q"]] = dict(ok=True, N=p["N"], n_points=p["n_points"], path=p["path"], waypoints=p["wps"], expansions=int(expansions[p["q"]]),
                               mid=p["mid"], points=p["points"], init_s=p["init_s"], final_s=p["final_s"], x0=p["x0"])
        back = []
    params = lbfgs_params or api.default_lbfgs_params(mem_size=16, past=3, delta=1e-6, g_epsilon=0.0, max_iterations=0, min_step=1e-32)
    launches0 = ctx.kernel_launches()
    results, rounds = ctx.optimize_lockstep([dict(N=p["N"], init_s=p["init_s"], final_s=p["final_s"], x0=p["x0"], points=p["points"])
                                             for p in back], params, max_in_flight)
    t4 = time.perf_counter()
    if stats is not None:
        stats.update(front_s=t1 - t0, points_s=t2 - t1, mid_s=t3 - t2, back_s=t4 - t3, rounds=int(rounds),
                     back_launches=ctx.kernel_launches() - launches0, back_problems=len(back))
    for p, r in zip(back, results):
        q = p["q"]
        out[q] = dict(ok=r["status"] >= 0, status=r["status"], N=p["N"], n_points=p["n_points"], path=p["path"], waypoints=p["wps"],
                      expansions=int(expansions[q]), mid=p["mid"], cost_at_warm_start=r["cost_at_start"], final_cost=float(r["final_cost"]),
                      iterations=int(r["iterations"]), evaluations=int(r["evaluations"]), T=r["T"], coeffs=r["coeffs"], x=r["x"],
                      seconds=float(r["seconds"]), points=p["points"])
    if certify:
        t5 = time.perf_counter()
        for p in back:
            r = out[p["q"]]
            r["clearance"] = certificate(ctx, r["T"], r["coeffs"])
        if stats is not None:
            stats["certify_s"] = time.perf_counter() - t5
    return out
