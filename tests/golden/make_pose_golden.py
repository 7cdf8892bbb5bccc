"""Write tests/golden/ref_pin_pose.npz: the REFERENCE'S OWN grad_cost_p (oracle/_ref/libref_pose_portable.so, built by
`make -C oracle ref` where the reference tree exists) at a set of sample poses, for the machines without the reference.

Cases: two maps (the reference's star map, map_star_pcd.npz at its resolution and threshold, half 8.5 = kernel_size 17 x 1.0 / 2 on
every axis; and a seeded five-layer map with half (3, 2, 0.5)) x every analytic shape and the Polygon x poly_params (0, 0, 0) and
(0.4, -0.3, 25).  Poses per case: seeded poses over and around the map; poses outside it on every side and beyond its z range;
boxes clipped at every face; yaws on a layer centre, between layers and far from all; voxels exactly at |p_rel_a| = half_a on each
axis; and (multi-layer map) safety_hor - sdf of one voxel below 0, at 0, in (0, mu] and above mu for the Circle.

    python tests/golden/make_pose_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import k3_points, oracle_py, ref_pose_py  # noqa: E402

SHAPES = ["star", "sdHorseshoe", "sdPie", "sdPie2", "sdArc", "sdTunnel", "sdCutDisk", "sdTrapezoid", "sdRhombus", "sdHeart",
          "sdRoundedX", "bigX", "sdRoundedCross", "sdOrientedVesica", "sdMoon", "sdUnevenCapsule", "Circle", "Polygon"]
PPS = [(0.0, 0.0, 0.0), (0.4, -0.3, 25.0)]
SAFETY = 0.7


def maps():
    g = np.load(os.path.join(HERE, "map_star_pcd.npz"))
    star = k3_points.gridmap_from_cloud(g["points"], float(g["occupancy_resolution"]), int(g["sta_threshold"]))
    rng = np.random.default_rng(20261017)
    occ = rng.random((30, 24, 5)) < 0.15
    occ[10:13, 10:13, :] = False
    occ[11, 11, 2] = True  # an isolated voxel, centre (6.5, -0.5, 0.0), for the exact cases
    return [("star", star.occ, star.boundary_min, star.res, (8.5, 8.5, 8.5)),
            ("multi", occ, np.array([-5.0, -12.0, -2.5]), 1.0, (3.0, 2.0, 0.5))]


def poses(occ, lo, res, half, name, shape, rng):
    size = np.array(occ.shape, dtype=np.float64)
    hi = lo + size * res
    zc = lo[2] + (np.arange(occ.shape[2]) + 0.5) * res
    out = [np.c_[rng.uniform(lo[0] - 4, hi[0] + 4, 24), rng.uniform(lo[1] - 4, hi[1] + 4, 24), rng.uniform(lo[2] - 1, hi[2] + 1, 24)]]
    mid = (lo + hi) / 2
    edge = []
    for a in range(2):  # outside each side, and boxes clipped at each face from inside
        for side, v in ((0, lo[a]), (1, hi[a])):
            p = mid.copy()
            p[a] = v + (12.0 if side else -12.0)
            edge.append(p.copy())
            p[a] = v + (-0.3 if side else 0.3)
            edge.append(p.copy())
    for yaw in (zc[0], zc[-1], (zc[0] + zc[1]) / 2, lo[2] - 20.0, hi[2] + 20.0):  # one layer, between layers, none
        edge.append(np.array([mid[0] + 0.25, mid[1] - 0.25, yaw]))
    out.append(np.array(edge))
    if name == "multi":
        c = np.array([6.5, -0.5, 0.0])  # the isolated voxel: |p_rel_a| = half_a exactly on each axis (yaw 0: p_rel = c - pos)
        out.append(np.array([c - [half[0], 0.0, 0.0], c + [half[0], 0.0, 0.0], c - [0.0, half[1], 0.0], c + [0.0, half[1], 0.0],
                             [c[0], c[1], c[2] - half[2]], [c[0], c[1], c[2] + half[2]]]))
        if shape == "Circle":  # the four smoothed-L1 regimes of that voxel (Circle at yaw 0: sdf = |p_rel| - radius)
            radius = -float(oracle_py.shape_sdf("Circle", np.zeros((1, 3)))[0])
            out.append(np.array([[c[0] - (radius + SAFETY - x), c[1], 0.0] for x in (-0.01, 0.0, 0.004, 0.3)]))
    return np.concatenate(out)


def main():
    assert ref_pose_py.available("portable"), "build oracle/_ref/libref_pose_portable.so first (make -C oracle ref)"
    rng = np.random.default_rng(7)
    out = {}
    case = []
    for mi, (name, occ, lo, res, half) in enumerate(maps()):
        out[f"map{mi}_occ"] = occ.astype(np.uint8)
        out[f"map{mi}_lo"] = np.asarray(lo, dtype=np.float64)
        out[f"map{mi}_res"] = np.float64(res)
        out[f"map{mi}_half"] = np.asarray(half, dtype=np.float64)
        for shape in SHAPES:
            for pi, pp in enumerate(PPS):
                P = poses(occ, np.asarray(lo, dtype=np.float64), res, half, name, shape, rng)
                rec = ref_pose_py.grad_cost_p(shape, pp, occ, lo, res, half, SAFETY, P)
                k = len(case)
                out[f"case{k}_poses"] = P
                out[f"case{k}_rec"] = rec
                case.append((mi, shape, pi))
    out["case_map"] = np.array([c[0] for c in case])
    out["case_shape"] = np.array([c[1] for c in case])
    out["case_pp"] = np.array([PPS[c[2]] for c in case])
    out["safety_hor"] = np.float64(SAFETY)
    path = os.path.join(HERE, "ref_pin_pose.npz")
    np.savez_compressed(path, **out)
    n = sum(out[f"case{k}_rec"].shape[0] for k in range(len(case)))
    act = sum(int((out[f"case{k}_rec"][:, 0] > 0).sum()) for k in range(len(case)))
    print(f"wrote {path}: {len(case)} cases, {n} poses, {act} active")


if __name__ == "__main__":
    main()
