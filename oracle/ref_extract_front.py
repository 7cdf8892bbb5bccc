"""Extract, VERBATIM, the reference's own source of the A* front end into oracle/_ref/front/gen/*.inc (git-ignored).

TEST INFRASTRUCTURE, the front-end counterpart of oracle/ref_extract.py (same `Source` cutter, same line-range guards).  The cut
definitions are the node test and the search of the reference's A*:
  * sw_manager.hpp: kernelConv<true/false>, visit_kernels_by_distance, checkKernelValue, checkSubSWCollision and the posEva2Rel
    it calls;
  * PCSmap_manager.h: or_mask, generateMapKernel2D, projInMap, getPointsInAABB2D;
  * GridMap3D.h / Gridmap3D.cpp: the GridMap3D members they call (toAddr, isInMap, isIndexValid, getGridIndex, getGridCubeCenter, isIndexOccupied,
    isIndexOccupiedFlate);
  * front_end_Astar.hpp: GridNode, the AstarPathSearcher class, and its initGridMap, reset, getHeu, getCustomCost, AstarGetSucc,
    AstarPathSearch and getPath.
`oracle/ref_front_shim.cpp` (ours) compiles them against the Eigen stand-in with storage-only stand-ins for the classes around
them.  Nothing generated here is committed: reference sources never enter the repository.

    python oracle/ref_extract_front.py [--ref /root/reference] [--out oracle/_ref/front/gen]
"""
from __future__ import annotations

import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_extract import Source  # noqa: E402


def extract(ref: str, out: str) -> None:
    os.makedirs(out, exist_ok=True)
    src = os.path.join(ref, "src")
    swm = Source(os.path.join(src, "swept_volume/include/swept_volume/sw_manager.hpp"))
    pcs = Source(os.path.join(src, "map_manager/include/map_manager/PCSmap_manager.h"))
    grid = Source(os.path.join(src, "map_manager/src/Gridmap3D.cpp"))
    gridh = Source(os.path.join(src, "map_manager/include/map_manager/GridMap3D.h"))
    ast = Source(os.path.join(src, "planner_algorithm/include/planner_algorithm/front_end_Astar.hpp"))

    files = {}
    # --- sw_manager.hpp: SweptVolumeManager members ---------------------------------------------------------------
    files["sw_front_methods.inc"] = "".join([
        swm.block(r"^\s*inline Eigen::Vector3d posEva2Rel\(", 0, expect_lines=(512, 530)),
        swm.block(r"^\s*inline bool kernelConv\(int kernel_i, const Eigen::Vector3i &ind\)", expect_lines=(1024, 1100)),
        swm.block(r"^\s*inline bool visit_kernels_by_distance\(", expect_lines=(1097, 1157)),
        swm.block(r"^\s*inline bool checkKernelValue\(double father_yaw,", expect_lines=(1154, 1170)),
        swm.block(r"^\s*inline bool checkSubSWCollision\(", expect_lines=(1167, 1212)),
    ])
    # --- PCSmap_manager.h: PCSmapManager members ------------------------------------------------------------------
    files["pcs_or_mask.inc"] = pcs.lines(r"^\s*static constexpr uint8_t or_mask\[8\]", r";", expect_lines=(30, 34))
    files["pcs_methods.inc"] = "".join([
        pcs.block(r"^\s*inline uint8_t\* generateMapKernel2D\(", expect_lines=(76, 109)),
        pcs.block(r"^\s*inline void projInMap\(", expect_lines=(124, 136)),
        pcs.block(r"^\s*inline void getPointsInAABB2D\(", expect_lines=(133, 159)),
    ])
    # --- GridMap3D.h / Gridmap3D.cpp: the in-class toAddr and the out-of-class GridMap3D definitions -----------------
    files["grid_toaddr.inc"] = gridh.block(r"^\s*inline int toAddr\(", expect_lines=(126, 131))
    files["grid_methods.inc"] = "".join([
        grid.block(r"^bool GridMap3D::isInMap\(", expect_lines=(40, 72)),
        grid.block(r"^bool GridMap3D::isIndexValid\(const Vector3i", expect_lines=(72, 104)),
        grid.block(r"^bool GridMap3D::isIndexValid\(\s*const int ix", expect_lines=(104, 136)),
        grid.block(r"^Vector3i GridMap3D::getGridIndex\(", expect_lines=(136, 178)),
        grid.block(r"^Vector3d GridMap3D::getGridCubeCenter\(int ix", expect_lines=(178, 183)),
        grid.block(r"^Vector3d GridMap3D::getGridCubeCenter\(const Vector3i", expect_lines=(183, 196)),
        grid.block(r"^bool GridMap3D::isIndexOccupied\(const Vector3i", expect_lines=(196, 212)),
        grid.block(r"^bool GridMap3D::isIndexOccupiedFlate\(", expect_lines=(212, 238)),
        grid.block(r"^bool GridMap3D::isIndexOccupied\(int ix", expect_lines=(238, 300)),
    ])
    # --- front_end_Astar.hpp ---------------------------------------------------------------------------------------
    files["astar_gridnode.inc"] = ast.block(r"^class GridNode\s*$", expect_lines=(10, 52), trailing_semicolon=True)
    files["astar_class.inc"] = ast.block(r"^class AstarPathSearcher\s*$", expect_lines=(52, 109), trailing_semicolon=True)
    files["astar_methods.inc"] = "".join([
        ast.block(r"^inline void AstarPathSearcher::initGridMap\(", expect_lines=(115, 153)),
        ast.block(r"^inline void AstarPathSearcher::reset\(", expect_lines=(153, 164)),
        ast.block(r"^inline double AstarPathSearcher::getHeu\(", expect_lines=(164, 183)),
        ast.block(r"^inline double AstarPathSearcher::getCustomCost\(", expect_lines=(184, 191)),
        ast.block(r"^inline void AstarPathSearcher::AstarGetSucc\(", expect_lines=(191, 242)),
        ast.block(r"^inline void AstarPathSearcher::AstarPathSearch\(", expect_lines=(242, 366)),
        ast.block(r"^inline vector<Vector3d> AstarPathSearcher::getPath\(", expect_lines=(366, 391)),
    ])

    for name, body in files.items():
        with open(os.path.join(out, name), "w", encoding="utf-8", errors="surrogateescape") as fh:
            fh.write("// GENERATED by oracle/ref_extract_front.py from the reference tree — verbatim reference source, do not commit.\n")
            fh.write(body)
    print(f"ref_extract_front: wrote {len(files)} fragments to {out}")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    ap.add_argument("--out", default=os.path.join(HERE, "_ref", "front", "gen"))
    a = ap.parse_args()
    if not os.path.isdir(a.ref):
        print("ref_extract_front: no reference tree at", a.ref, file=sys.stderr)
        sys.exit(2)
    extract(a.ref, a.out)
