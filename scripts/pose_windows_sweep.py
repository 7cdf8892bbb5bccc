"""Device time of one cost + gradient evaluation with and without the layer-3 pose windows (SVSDF_FORCE_POSE_WINDOWS = 1 / 2), over
the number of query points, on config 2's trajectory (8 pieces, K1 = 134) and on a 64-piece, 299.84 s one (K1 = 1999): the
measurement behind the layer-3 rule of pose_windows() in csrc/svsdf_runtime_eval.cpp.

    python scripts/pose_windows_sweep.py [--repeats R] [--rounds K] [--out FILE]

Prints one JSON line per (trajectory, P): the median over K alternating rounds of R back-to-back evaluations per setting.
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from implicit_svsdf_planner_b200 import api, scenes
    import make_outer_edges_golden as mko

    sc = scenes.make_scene("star", 8, 200_000)
    _, T64, co64, _ = mko.scene("long64")
    cases = [("config2", sc.T, sc.coeffs_colmajor(), sc.points, P) for P in (1_000, 4_000, 16_000, 64_000, 200_000)]
    pts64 = mko.long64_points(400_000, 7)
    cases += [("long64", T64, co64, pts64, P) for P in (25_000, 100_000, 200_000, 400_000)]
    lines = []
    for name, T, co, pts, P in cases:
        ms = {"1": [], "2": []}
        ctxs = {}
        for w in ("1", "2"):
            os.environ["SVSDF_FORCE_POSE_WINDOWS"] = w  # read when the context is created
            c = api.Context("star", strict_fp=True)
            c.set_points(pts[:P])
            c.cost_grad_device(T, co, repeats=2, fetch=False)  # warm-up
            ctxs[w] = c
        for _ in range(args.rounds):
            for w in ("1", "2"):
                ms[w].append(ctxs[w].cost_grad_device(T, co, repeats=args.repeats, fetch=False)[0])
        for c in ctxs.values():
            c.close()
        m1, m2 = statistics.median(ms["1"]), statistics.median(ms["2"])
        K1 = len(mko.lattice(float(np.sum(T))))
        line = dict(traj=name, P=P, K1=K1, layer3_records=(K1 + 1) * 22 * 21, layer3_samples=21 * P, ms_layer2=m1, ms_layers23=m2,
                    gain=1.0 - m2 / m1, runs_layer2=ms["1"], runs_layers23=ms["2"])
        print(json.dumps(line), flush=True)
        lines.append(line)
    os.environ.pop("SVSDF_FORCE_POSE_WINDOWS", None)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(lines, fh, indent=1)


if __name__ == "__main__":
    main()
