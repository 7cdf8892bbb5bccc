"""Generate tests/golden/ref_pin_scale_edges.npz: what THE REFERENCE'S OWN CODE, built with its `useScale` switch on, returns
on the edge scenes of the outer solve and of the interior branch under schedules at the limits of what svsdf_set_scale
accepts.

    make -C oracle ref && python tests/golden/make_scale_edges_golden.py [out.npz]     (needs the reference tree)

The trajectories are the rigid edge scenes (tests/golden/make_outer_edges_golden.py, make_gsip_edges_golden.py), imported,
not copied.  Schedules (a_x, a_y, b_x, b_y, w_x, w_y, phi_x, phi_y):
  example     the reference's commented example
  limit_w     a = 1, b = +-0.3, |w| 300 + |phi| just under 1e6 (phi_y beyond pi, w_y and b_y negative): on long64 the sin
              argument sweeps up to 9.98e5 rad, the top of the Cody-Waite reduction
  fast        w of 250 and -310 rad/s: S changes within one descent step (0.01 s): long descents, accepted halvings up to j = 28
  thin        s_y = 1 - 0.999999 sin(pi/2) = 1.00000000003e-6 at every t (w_y = 0), the smallest scale svsdf_set_scale
              accepts: St^-1 = 1e6 on y; x varies (w_x < 0, |phi_x| > pi)
  needle      constant a = (40, 0.025), b = w = 0: a parked robot stays exactly flat in t
  zero_phase  b != 0, w = 0, phi = 0, a = 1: sin(0) = 0, S = I exactly, the rigid kernels' arithmetic
  pi_phase    b = (0.95, -0.95), w = 0, phi = (pi, 3 pi), a = 1: sin(phi) ~ 1e-16, S differs from I in the last bits only

Matrix (trajectory: schedules), chosen so that every branch the scaled code changes is reached under a schedule; which
branch each pair reaches is asserted by tests/test_oracle_scale_edges.py:
  tiny_k1        example, thin
  tiny_n2        example, limit_w, fast, thin, pi_phase
  long64         example, limit_w
  parked         example, fast, needle, zero_phase
  broken         example, limit_w, fast, zero_phase
  junction       example, thin
  endpoints      example, limit_w, thin, zero_phase
  midstop        example, fast, needle, pi_phase
  circle_static  example, needle, pi_phase
  circle_spin    example, fast
  spin           fast, zero_phase (the outer-edge scene whose first points' rigid descents stop at the 1000-iteration
                 cap: under zero_phase they reach it through the scaled kernels; "fast" alone reaches deep halvings, but
                 no trajectory here reaches the cap under it)

Stored per trajectory: the inputs (long64 thinned like ref_pin_outer_edges.npz); per (trajectory, schedule) and variant
("portable": the reference with its per-sample sin/cos/atan2 redirected to the pinned algorithms the oracle's default build and
the strict kernels implement; "glibc": as it runs on x86-64): RefPath.query's sdf, t* and gradient, and for "portable" also
query_outer's.  Written with fixed zip timestamps, so regenerating gives the same bytes.  Only outputs enter the file.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import make_gsip_edges_golden as mkg  # noqa: E402
import make_outer_edges_golden as mko  # noqa: E402
from make_scale_golden import save_npz_fixed  # noqa: E402

OUT = os.path.join(HERE, "ref_pin_scale_edges.npz")
PI = np.pi
SCHEDULES = {
    "example": (0.8, 0.8, 0.6, 0.4, 1.5, 1.8, -1.0, 0.0),
    "limit_w": (1.0, 1.0, 0.3, -0.3, 3333.33, -3333.0, 0.5, -4.0),
    "fast": (1.0, 0.9, 0.4, -0.3, 250.0, -310.0, 0.3, 2.0),
    "thin": (0.8, 1.0, 0.5, -0.999999, -1.3, 0.0, 7.0, PI / 2),
    "needle": (40.0, 0.025, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0),
    "zero_phase": (1.0, 1.0, 0.3, -0.2, 0.0, 0.0, 0.0, 0.0),
    "pi_phase": (1.0, 1.0, 0.95, -0.95, 0.0, 0.0, PI, 3 * PI),
}
MATRIX = {
    "tiny_k1": ("example", "thin"),
    "tiny_n2": ("example", "limit_w", "fast", "thin", "pi_phase"),
    "long64": ("example", "limit_w"),
    "parked": ("example", "fast", "needle", "zero_phase"),
    "broken": ("example", "limit_w", "fast", "zero_phase"),
    "junction": ("example", "thin"),
    "endpoints": ("example", "limit_w", "thin", "zero_phase"),
    "midstop": ("example", "fast", "needle", "pi_phase"),
    "circle_static": ("example", "needle", "pi_phase"),
    "circle_spin": ("example", "fast"),
    "spin": ("fast", "zero_phase"),
}
OUTER_SCENES = ("tiny_k1", "tiny_n2", "long64", "parked", "broken", "junction", "spin")
VARIANTS = ("glibc", "portable")


def pairs():
    return [(t, s) for t, ss in MATRIX.items() for s in ss]


def scene(name):
    """(shape, T, coeffs column-major, points P x 3) of one trajectory as the fixture stores it."""
    if name in OUTER_SCENES:
        return mko.golden_scene(name)
    return mkg.scene(name)


def generate(path=OUT):
    from oracle import scale_py

    out = {"schedules": np.array(list(SCHEDULES)), "sched_values": np.array(list(SCHEDULES.values()))}
    for name, scheds in MATRIX.items():
        shape, T, co, pts = scene(name)
        out.update({f"{name}_shape": np.array(shape), f"{name}_T": T, f"{name}_coeffs": co, f"{name}_points": pts})
        for sk in scheds:
            for v in VARIANTS:
                ref = scale_py.RefScaled(shape, sched=SCHEDULES[sk], threads=8, variant=v)
                ref.set_traj(T, co)
                key = f"{name}_{sk}_{v}"
                out[key + "_sdf"], out[key + "_tstar"], out[key + "_grad"] = ref.query(pts)
                if v == "portable":
                    out[key + "_osdf"], out[key + "_otstar"], out[key + "_ograd"] = ref.query_outer(pts)
            print(name, sk, "points", len(pts), "inside", int((out[f"{name}_{sk}_portable_osdf"] <= 0).sum()))
    save_npz_fixed(path, out)
    return path


if __name__ == "__main__":
    p = generate(sys.argv[1] if len(sys.argv) > 1 else OUT)
    print(p, os.path.getsize(p), "bytes")
