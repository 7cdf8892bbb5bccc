"""Generate tests/golden/ref_pin_gsip_edges.npz: what THE REFERENCE'S OWN CODE returns on the edge scenes of the interior
(GSIP) branch of getTrueSDFofSweptVolume<true>.

    make -C oracle ref_path && python tests/golden/make_gsip_edges_golden.py      (needs the reference's sources)

The scenes reach the parts of the branch that ordinary scenes barely touch:
  endpoints      points inside the robot's footprint at the start and at the end pose of the star trajectory: t* lands where
                 the robot is at rest, so the velocity fallback scans forward (t* < 0.1) or backward (t* > D - 0.1)
  midstop        a two-piece quintic, written by hand, that comes to a full stop at its junction: t* in the middle of the
                 trajectory with |v| < 0.01 (no scan, the ring starts from the direction of a tiny velocity); also reaches the
                 9-round cap of the ring search
  circle_static  a Circle (radius 1) parked at the origin for the whole trajectory (N = 2): points on the boundary (outer sdf
                 exactly 0.0, which `!(sdf > 0)` sends inside), inside and at the centre (all ring samples tie); the scan runs
                 to the end without finding motion and the ring origin is atan2(0, -0)
  circle_spin    the same Circle spinning in place (x, y constant, yaw linear): |v| = |yaw rate| >= 0.01, vx = vy = 0

Stored per scene and variant ("portable": the reference with sin/cos/atan2 redirected to the pinned fdlibm algorithm the
oracle's default build and the strict CUDA kernels implement; "glibc": the reference as it runs on x86-64): the inputs,
RefPath.query (sdf, t*, gradient) and RefPath.query_outer (sdf, t*, gradient).  The input builders are shared with the
tests (tests/test_oracle_ref_pin.py, tests/test_gpu_gsip.py), which import this module.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "ref_pin_gsip_edges.npz")
SCENES = ("endpoints", "midstop", "circle_static", "circle_spin")
VARIANTS = ("glibc", "portable")


def colmajor(C):
    """[piece][dim][power] coefficients -> the 6N x 3 column-major buffer of the C ABI (offset d * 6N + 6i + k)."""
    C = np.asarray(C, dtype=np.float64)
    return np.ascontiguousarray(C.transpose(1, 0, 2)).reshape(-1)


def _disc(rng, centre, radius, n):
    a = rng.uniform(0.0, 2.0 * np.pi, n)
    r = radius * np.sqrt(rng.uniform(0.0, 1.0, n))
    return np.c_[centre[0] + r * np.cos(a), centre[1] + r * np.sin(a), np.zeros(n)]


def _rest_to_rest(a, b, T):
    """Quintic from a to b in time T with zero velocity and acceleration at both ends (ascending powers)."""
    d = b - a
    return np.array([a, 0.0, 0.0, 10.0 * d / T**3, -15.0 * d / T**4, 6.0 * d / T**5])


def _circle_points():
    ang = np.arange(16) * (np.pi / 8)
    ring = np.c_[np.cos(ang), np.sin(ang)]
    ring[[0, 4, 8, 12]] = [[1.0, 0.0], [0.0, 1.0], [-1.0, 0.0], [0.0, -1.0]]  # exactly on the boundary: outer sdf 0.0
    half = 0.5 * ring[1::2]
    xy = np.r_[ring, half, [[0.0, 0.0], [0.3, 0.2], [-0.75, 0.0], [0.0, 0.999]]]
    return np.c_[xy, np.zeros(len(xy))]


def scene(name):
    """(shape, T, coeffs column-major, points P x 3) of one edge scene."""
    sys.path.insert(0, ROOT)
    from implicit_svsdf_planner_b200 import scenes

    if name == "endpoints":
        init_s, final_s, q, T = scenes.make_trajectory("star", 8)
        b = scenes.minco_dense(init_s, final_s, q, T)
        rng = np.random.default_rng(11)
        pts = np.r_[_disc(rng, init_s[:2, 0], 2.5, 60), _disc(rng, final_s[:2, 0], 2.5, 60)]
        return "star", T, np.ascontiguousarray(b.T).reshape(-1), pts
    if name == "midstop":
        T = np.array([2.0, 2.0])
        C = np.zeros((2, 3, 6))
        C[0, 0] = _rest_to_rest(0.0, 5.0, 2.0)           # piece 0: along x, yaw 0, stops at (5, 0)
        C[1, 0, 0] = 5.0
        C[1, 1] = _rest_to_rest(0.0, 4.0, 2.0)           # piece 1: along y while turning to yaw pi / 2
        C[1, 2] = _rest_to_rest(0.0, np.pi / 2, 2.0)
        rng = np.random.default_rng(12)
        return "star", T, colmajor(C), _disc(rng, (5.0, 0.0), 2.5, 60)
    if name == "circle_static":
        return "Circle", np.array([1.0, 1.0]), colmajor(np.zeros((2, 3, 6))), _circle_points()
    if name == "circle_spin":
        C = np.zeros((2, 3, 6))
        C[0, 2, 1] = 0.5                                 # yaw = 0.5 t
        C[1, 2, 0], C[1, 2, 1] = 0.5, 0.5
        return "Circle", np.array([1.0, 1.0]), colmajor(C), _circle_points()
    raise KeyError(name)


def main():
    sys.path.insert(0, ROOT)
    from oracle import ref_py as R

    if not R.available("portable"):
        R.build()
    out = {}
    for name in SCENES:
        shape, T, co, pts = scene(name)
        out.update({f"{name}_shape": shape, f"{name}_T": T, f"{name}_coeffs": co, f"{name}_points": pts})
        for v in VARIANTS:
            ref = R.RefPath(shape, threads=8, variant=v)
            ref.set_traj(T, co)
            out[f"{name}_sdf_{v}"], out[f"{name}_tstar_{v}"], out[f"{name}_grad_{v}"] = ref.query(pts)
            out[f"{name}_osdf_{v}"], out[f"{name}_otstar_{v}"], out[f"{name}_ograd_{v}"] = ref.query_outer(pts)
            print(name, v, "points", len(pts), "inside", int((out[f"{name}_sdf_{v}"] <= 0).sum()))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
