"""Generate tests/golden/ref_pin_scale.npz: outputs of THE REFERENCE'S OWN CODE for a deformable robot.

    make -C oracle ref && python tests/golden/make_scale_golden.py [out.npz]     (only where the reference tree exists)

oracle/_ref/libref_path_scaled_{glibc,portable}.so are the reference's source (oracle/ref_extract_scale.py,
oracle/ref_path_scaled_shim.cpp): its `useScale` switch turned on and this project's schedule supplying getScale(t) =
diag(a_x + sin(w_x t + phi_x) b_x, a_y + sin(w_y t + phi_y) b_y, 1).  For every registry shape, Circle and the Polygon
fallback, two body-frame pre-transforms and three schedules (the reference's commented example, a constant anisotropic
scale, the identity) the fixture holds getTrueSDFofSweptVolume's sdf, t* and gradient per point (outside and interior
points), and for the star the accumulating penalty loop (cost, gradT, gradC).  The file is written with fixed zip
timestamps, so regenerating it gives the same bytes.
"""
import io
import os
import sys
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from implicit_svsdf_planner_b200 import scenes  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "ref_pin_scale.npz")
SHAPES = ["star", "sdHorseshoe", "sdPie", "sdPie2", "sdArc", "sdTunnel", "sdCutDisk", "sdTrapezoid", "sdRhombus", "sdHeart",
          "sdRoundedX", "bigX", "sdRoundedCross", "sdOrientedVesica", "sdMoon", "sdUnevenCapsule", "Circle", "fallbackPolygon"]
PRE = [(0.0, 0.0, 0.0), (0.3, -0.2, 25.0)]
# (a_x, a_y, b_x, b_y, w_x, w_y, phi_x, phi_y)
SCHEDULES = {
    "example": (0.8, 0.8, 0.6, 0.4, 1.5, 1.8, -1.0, 0.0),  # sw_manager.hpp:498-500
    "aniso": (1.3, 0.7, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0),     # constant anisotropic scale (b = 0)
    "identity": (1.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0),
}
VARIANTS = ("glibc", "portable")  # reference variant; the oracle's "glibc" / "default" must match it


def scene():
    """A 6-piece star scene with a narrow corridor: outside points and a few interior ones for every shape."""
    sc = scenes.make_scene("star", 6, 80, clearance=2.35)
    return sc.T, sc.coeffs_colmajor(), np.ascontiguousarray(sc.points[:, :2]), (sc.weight_p, sc.safety_hor, sc.rho)


def save_npz_fixed(path, arrays):
    """np.savez with a fixed timestamp on every member (np.savez stamps the current time)."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            zi = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            zi.external_attr = 0o644 << 16
            zf.writestr(zi, buf.getvalue())


def generate(path=OUT):
    from oracle import scale_py

    T, co, pts, (wp, sh, rho) = scene()
    pts0 = np.c_[pts, np.zeros(len(pts))]
    out = {"T": T, "coeffs": co, "points": pts, "params": np.array([wp, sh, rho]), "shapes": np.array(SHAPES),
           "pre": np.array(PRE), "schedules": np.array(list(SCHEDULES)), "sched_values": np.array(list(SCHEDULES.values()))}
    for v in VARIANTS:
        for sk, sv in SCHEDULES.items():
            for ip, pp in enumerate(PRE):
                for s in SHAPES:
                    ref = scale_py.RefScaled(s, sched=sv, poly_params=pp, weight_p=wp, safety_hor=sh, rho=rho, threads=8, variant=v)
                    ref.set_traj(T, co)
                    sdf, ts, g = ref.query(pts0)
                    out[f"{v}_{sk}_{ip}_{s}_sdf"], out[f"{v}_{sk}_{ip}_{s}_tstar"], out[f"{v}_{sk}_{ip}_{s}_grad"] = sdf, ts, g
            # one thread: the loop adds its points in a critical section, in whatever order the threads reach it
            ref = scale_py.RefScaled("star", sched=sv, weight_p=wp, safety_hor=sh, rho=rho, threads=1, variant=v)
            ref.set_points(pts)
            cost, gT, gC = ref.cost_grad(T, co)
            out[f"{v}_{sk}_cost"], out[f"{v}_{sk}_gradT"], out[f"{v}_{sk}_gradC"] = np.float64(cost), gT, gC
    save_npz_fixed(path, out)
    return path


if __name__ == "__main__":
    p = generate(sys.argv[1] if len(sys.argv) > 1 else OUT)
    g = np.load(p)
    print(p, len(g.files), "arrays; interior points (portable, example, star):", int((g["portable_example_0_star_sdf"] <= 0).sum()))
