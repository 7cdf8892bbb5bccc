"""What the reference's compiled code returns on the seeded inputs of the tests that compare against it at scale
(tests/test_oracle_ref_pin.py, test_oracle_mesh.py, test_oracle_mid.py, test_gpu_ref_pin.py) -> tests/golden/ref_live.npz, so that
those comparisons run wherever the repository does.

    make -C oracle ref && python tests/golden/make_live_golden.py      (needs the reference's sources for `make ref`)

The tests compare large per-point outputs bit for bit, so those are stored as SHA-256 digests of their float64 bytes (the digest is the
whole comparison, and 1e5 points x 18 shapes would not fit a small fixture); small outputs are stored as arrays.  The input generators
below are shared with the tests."""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "ref_live.npz")
PRE = [(0.0, 0.0, 0.0), (-0.4, 0.15, -70.0)]  # body-frame pre-transforms of the 1e5-point shape comparison
FWN_MESHES = ["synthetic_star", "two_faces", "seven_faces", "grid_900", "degenerate_duplicates"]
MID_NS = (4, 9)
MID_DRAWS = 3


def digest(a, signed_zero=True):
    """SHA-256 of the float64 bytes; signed_zero=False maps -0.0 to +0.0 first."""
    a = np.ascontiguousarray(a, dtype=np.float64).ravel()
    if not signed_zero:
        a = a + 0.0
    return hashlib.sha256(a.tobytes()).hexdigest()


def shape_points(n=100_000):
    rng = np.random.default_rng(77)
    return np.c_[rng.uniform(-9.0, 9.0, (n, 2)), rng.uniform(-1.0, 1.0, n)]


def fwn_mesh(mesh):
    """(V, F, Q) of the winding-number comparison: meshes that exercise every branch of the builder (2 items, the exhaustive <= 6
    split, the sorted <= 32 split, the 16-span binning, coincident centres) and 3000 queries around each."""
    sys.path.insert(0, ROOT)
    from implicit_svsdf_planner_b200 import scenes

    rng = np.random.default_rng(9)
    if mesh == "synthetic_star":
        V, F = scenes.extrude_outline(scenes.star_outline(n_per_edge=4))
    elif mesh in ("two_faces", "seven_faces"):
        nf = 2 if mesh == "two_faces" else 7
        V = rng.uniform(-2, 2, size=(3 * nf, 3))
        F = np.arange(3 * nf, dtype=np.int32).reshape(nf, 3)
    elif mesh == "grid_900":
        n = 16
        xs, ys = np.meshgrid(np.linspace(-3, 3, n), np.linspace(-2, 2, n))
        V = np.c_[xs.ravel(), ys.ravel(), 0.3 * np.sin(xs.ravel() * 2.0) * np.cos(ys.ravel())]
        F = []
        for i in range(n - 1):
            for j in range(n - 1):
                a = i * n + j
                F += [[a, a + 1, a + n + 1], [a, a + n + 1, a + n]]
        F = np.asarray(F, dtype=np.int32)
    else:  # many faces sharing one centre: the span partition cannot split them
        base = rng.uniform(-1, 1, size=(3, 3))
        V = np.concatenate([base * (1.0 + 0.0 * k) for k in range(40)] + [rng.uniform(-2, 2, size=(30, 3))])
        F = np.arange(len(V), dtype=np.int32).reshape(-1, 3)
    lo, hi = V.min(axis=0) - 1.5, V.max(axis=0) + 1.5
    Q = np.zeros((3000, 3))
    Q[:, :2] = rng.uniform(lo[:2], hi[:2], size=(3000, 2))
    Q[1500:] = rng.uniform(lo, hi, size=(1500, 3))
    return V, F, Q


def mid_draws():
    """(key, N, config overrides, (init_s, final_s, Q, rots), x): three perturbed x per problem and parameter set."""
    import make_mid_golden as mk

    rng = np.random.default_rng(3)
    for N in MID_NS:
        init_s, final_s, Q, rots, x = mk.problem(N, 500 + N)
        for cname, over in mk.CONFIGS.items():
            for k in range(MID_DRAWS):
                yield f"mid_{N}_{cname}_{k}", N, over, (init_s, final_s, Q, rots), x + rng.normal(0, 0.2, x.shape)


def gpu_scene():
    from implicit_svsdf_planner_b200 import scenes

    return scenes.make_scene("star", 8, 20_000, seed_map=991)


def main():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    import make_fwn_golden as mf

    from implicit_svsdf_planner_b200 import api
    from oracle import ref_py as R

    out = {}
    shapes = [str(s) for s in np.load(os.path.join(HERE, "ref_pin_shapes.npz"))["shapes"]]
    rel = shape_points()
    for rv in ("glibc", "portable"):
        for ip, pp in enumerate(PRE):
            for s in shapes:
                out[f"shape_sdf_{rv}_{ip}_{s}"] = np.str_(digest(R.shape_sdf(s, rel, pp, variant=rv)))
        for s in shapes:
            out[f"shape_grad1_{rv}_{s}"] = np.str_(digest(R.shape_grad1(s, rel[:5000], variant=rv)))
    for mesh in FWN_MESHES:
        V, F, Q = fwn_mesh(mesh)
        rc, rd = mf.ref_fwn_tree(V, F)
        out[f"fwn_{mesh}_w"] = mf.ref_fwn(V, F, Q)
        out[f"fwn_{mesh}_children"], out[f"fwn_{mesh}_data"] = rc, rd
    for key, N, over, prob, xx in mid_draws():
        cfg = api.mid_default_config(**over)
        i_s, f_s, q, r, _ = api._mid_args(*prob)
        cr, gr = R.mid_cost(cfg, N, i_s, f_s, q, r, xx)
        out[key + "_x"], out[key + "_cost"], out[key + "_grad"] = xx, np.float64(cr), gr
    sc = gpu_scene()
    ref = R.RefPath("star", weight_p=sc.weight_p, safety_hor=sc.safety_hor, rho=sc.rho, threads=os.cpu_count() or 8, variant="portable")
    ref.set_traj(sc.T, sc.coeffs_colmajor())
    for name, a in zip(("sdf", "tstar", "grad"), ref.query(np.c_[sc.points[:, :2], np.zeros(sc.P)])):
        out[f"gpu20k_{name}"] = np.str_(digest(a, signed_zero=False))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes,", len(out), "entries")


if __name__ == "__main__":
    main()
