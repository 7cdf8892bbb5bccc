"""One whole plan on the reference's own star scene (pcds/map_star.pcd + pcds/trajectory_star.txt + config/star.yaml, carried as
tests/golden/map_star_pcd.npz): point cloud -> map -> A* front end -> waypoints / query points -> mid-end warm start -> SVSDF back end.
Prints one JSON line.  Needs an H100:  python scripts/run_plan.py [--shape star]"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from implicit_svsdf_planner_b200 import api, plan, scenes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="star")
    args = ap.parse_args()
    g = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "map_star_pcd.npz"))
    cmap = plan.gridmap3d_from_cloud(g["points"], float(g["occupancy_resolution"]), int(g["sta_threshold"]))
    ctx = api.Context(args.shape, weight_p=scenes.YAML["weight_p"], safety_hor=scenes.YAML["safety_hor"], rho=scenes.YAML["rho"])
    t0 = time.perf_counter()
    r = plan.generate_traj(ctx, cmap, g["start"][:2], g["end"][:2], kernel_size=int(g["kernel_size"]), traj_parlength=float(g["traj_parlength"]))
    dt = time.perf_counter() - t0
    out = {k: v for k, v in r.items() if k not in ("path", "waypoints", "coeffs", "x", "T", "mid")}
    if r.get("ok"):
        out.update(path_nodes=int(len(r["path"])), total_duration=float(np.sum(r["T"])), mid=dict(status=r["mid"]["status"], cost=r["mid"]["cost"], iterations=r["mid"]["iterations"]))
    out.update(scene="reference pcds/map_star.pcd, trajectory_star.txt, config/star.yaml", occupied_voxels=int(cmap.occ.sum()), map_size=list(cmap.occ.shape),
               wall_seconds=dt)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
