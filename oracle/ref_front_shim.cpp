// oracle/ref_front_shim.cpp — TEST INFRASTRUCTURE: the REFERENCE'S OWN SOURCE of the A* front end, compiled where it lies.
//
// Builds oracle/_ref/libref_front_<variant>.so (git-ignored; `make -C oracle ref`, only where the reference tree exists):
//   * the shape classes and BasicShape::initShape: oracle/ref_shape_scaffold.inc over the fragments of oracle/ref_extract.py,
//     exactly as in libref_path_*;
//   * the node test and the search: oracle/_ref/front/gen/*.inc, cut VERBATIM by oracle/ref_extract_front.py —
//     SweptVolumeManager::posEva2Rel / kernelConv / visit_kernels_by_distance / checkKernelValue / checkSubSWCollision,
//     PCSmapManager::generateMapKernel2D / projInMap / getPointsInAABB2D, the GridMap3D members they call, GridNode, the
//     AstarPathSearcher class and its initGridMap / reset / getHeu / getCustomCost / AstarGetSucc / AstarPathSearch / getPath;
//   * ros::Time / ROS_WARN / ROS_ERROR: oracle/ref_shim/ros/time_stub.hpp.
// What is OURS here is storage only — the members of GridMap3D, PCSmapManager and SweptVolumeManager that the cut methods read
// (sizes, bounds, resolution, the occupancy array, the packed map kernel) — plus the C API at the bottom.  Two choices:
//   * The map is the product's: X x Y cells of size res from (ox, oy), boundary_xyzmax = (ox + X res, oy + Y res), one z layer
//     [0, res] (every query has z = 0).
//   * SweptVolumeManager::isIndexValid / isIndexOccupied have EMPTY bodies in the reference (sw_manager.hpp:1026-1031: falling off
//     the end of a bool function), so kernelConv<false> is undefined there as written; here they forward to GridMap3D's.
//   * generateMapKernel2D's buffer is copied into one with a zero byte of slack: kernelConv<true> reads one byte past the last row
//     (sw_manager.hpp:1087); that byte only feeds bits the byte kernel masks out.
//
// Variants (oracle/Makefile): glibc (the reference as it runs on x86-64) and portable (-DREF_LIBM_PORTABLE: every sin/cos/atan2 in the
// reference text — AngleAxisd's in checkSubSWCollision and initShape, the shapes' constants — is the pinned fdlibm algorithm the
// CUDA kernels implement, as in libref_path_portable).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <map>
#include <memory>
#include <queue>
#include <sstream>
#include <string>
#include <vector>

#ifdef REF_LIBM_PORTABLE
#include "portable_sincos.hpp"
namespace ref_libm {
inline double psin(double x) { double s, c; oracle::psc::sincos(x, s, c); return s; }
inline double pcos(double x) { double s, c; oracle::psc::sincos(x, s, c); return c; }
inline double patan2(double y, double x) { return oracle::psc::atan2(y, x); }
}  // namespace ref_libm
namespace std {
using ref_libm::patan2;
using ref_libm::pcos;
using ref_libm::psin;
}  // namespace std
using ref_libm::patan2;
using ref_libm::pcos;
using ref_libm::psin;
#define REF_SHIM_SIN(x) ref_libm::psin(x)
#define REF_SHIM_COS(x) ref_libm::pcos(x)
#endif

#include <Eigen/Eigen>
#include "ros/time_stub.hpp"

#ifdef REF_LIBM_PORTABLE
#define sin psin
#define cos pcos
#define atan2 patan2
#endif

using namespace Eigen;  // utils/config.hpp:10
using namespace std;    // utils/config.hpp:11

struct Config {  // utils/config.hpp: the fields the front end reads
    vector<double> poly_params{0.0, 0.0, 0.0};
    int kernel_yaw_num{18};
    int kernel_size{17};
    double occupancy_resolution{1.0};
    double front_end_safeh{0.0};
};

#include "ref_shape_scaffold.inc"  // BasicShape + initShape + the shape classes (Shape.hpp), as in libref_path_*
#include "_ref/gen/sw_macros.inc"  // TRAJ_ORDER, useScale, useNumer, pi (sw_manager.hpp:16-20)

class GridMap3D {  // storage of GridMap3D.h:133-151; the methods are Gridmap3D.cpp's
  public:
    bool isInMap(const Vector3d &pos_w) const;
    bool isIndexValid(const Vector3i &index) const;
    bool isIndexValid(const int ix, const int iy, const int iz) const;
    bool isIndexOccupied(int ix, int iy, int iz);
    bool isIndexOccupied(const Vector3i &index);
    bool isIndexOccupiedFlate(const Vector3i &index, const int flate_pix);
    Vector3i getGridIndex(const Vector3d &pos_w);
    Vector3d getGridCubeCenter(const Vector3i &index);
    Vector3d getGridCubeCenter(int ix, int iy, int iz);
#include "_ref/front/gen/grid_toaddr.inc"
    int X_size{0}, Y_size{0}, Z_size{0}, totalsize{0};
    Vector3d boundary_xyzmin, boundary_xyzmax;
    double grid_resolution{1.0};
    std::vector<double> grid_map_store;
    double *grid_map{nullptr};
    typedef shared_ptr<GridMap3D> Ptr;
};
#include "_ref/front/gen/grid_methods.inc"

class PCSmapManager {  // storage of PCSmap_manager.h:221-239
  public:
#include "_ref/front/gen/pcs_or_mask.inc"
#include "_ref/front/gen/pcs_methods.inc"
    Vector3d boundary_xyzmin, boundary_xyzmax;
    double occupancy_resolution{1.0};
    GridMap3D::Ptr occupancy_map;
    uint8_t *mk{nullptr};
    typedef shared_ptr<PCSmapManager> Ptr;
};

class SweptVolumeManager {  // storage of sw_manager.hpp:129-153
  public:
    uint8_t *map_kernel{nullptr};
    int map_Xsize{0}, map_Ysize{0}, map_Zsize{0};
    Config config;
    int kernel_count{0};
    int kernelsize{0};
    BasicShape *current_robot_shape{nullptr};
    GridMap3D *grid{nullptr};
    // sw_manager.hpp:1026-1031 leave these empty; see the header comment
    bool isIndexValid(const int ix, const int iy, const int iz) const { return grid->isIndexValid(ix, iy, iz); }
    bool isIndexOccupied(int ix, int iy, int iz) { return grid->isIndexOccupied(ix, iy, iz); }
#include "_ref/front/gen/sw_front_methods.inc"
    typedef shared_ptr<SweptVolumeManager> Ptr;
};

struct SE3State;  // named by a declaration of AstarPathSearcher that is never defined here (getastarSE3Path)
#include "_ref/front/gen/astar_gridnode.inc"
#include "_ref/front/gen/astar_class.inc"
#include "_ref/front/gen/astar_methods.inc"

#ifdef REF_LIBM_PORTABLE
#undef sin
#undef cos
#undef atan2
#endif
#undef pi

// =====================================================================================================================
// C API (ours)
// =====================================================================================================================
namespace {
struct Quiet {  // initShape / initGridMap print
    std::streambuf *old;
    std::ostringstream sink;
    Quiet() : old(std::cout.rdbuf(sink.rdbuf())) {}
    ~Quiet() { std::cout.rdbuf(old); }
};

BasicShape *make_shape(const std::string &n, const Config &conf) {  // the registry of sw_manager.hpp:187-235
#define REF_SHAPE(N) if (n == #N) return new N(conf);
    REF_SHAPE(sdUnevenCapsule) REF_SHAPE(sdCutDisk) REF_SHAPE(sdTrapezoid) REF_SHAPE(sdRhombus) REF_SHAPE(star)
    REF_SHAPE(sdTunnel) REF_SHAPE(sdHorseshoe) REF_SHAPE(sdHeart) REF_SHAPE(sdOrientedVesica) REF_SHAPE(sdRoundedCross)
    REF_SHAPE(sdRoundedX) REF_SHAPE(bigX) REF_SHAPE(sdMoon) REF_SHAPE(sdPie) REF_SHAPE(sdPie2) REF_SHAPE(sdArc)
    REF_SHAPE(Circle)
#undef REF_SHAPE
    return nullptr;
}

struct Front {
    Config conf;
    std::unique_ptr<BasicShape> shape;
    GridMap3D::Ptr grid;
    PCSmapManager::Ptr env;
    SweptVolumeManager::Ptr sv;
    AstarPathSearcher astar;
    std::vector<uint8_t> kernel_bytes;  // generateMapKernel2D's output + 1 zero byte
    int mk_len{0};
};
}  // namespace

extern "C" {

const char *rf_variant() {
#ifdef REF_LIBM_PORTABLE
    return "portable";
#else
    return "glibc";
#endif
}

// One front end: shape (+ pre-transform), kernels (ks, K, res, safeh) and the map occ [X][Y] (0/1) at origin (ox, oy), cell res.
// NULL for an unknown shape name.
void *rf_create(const char *name, const double *poly_params, int ks, int K, double res, double safeh, const uint8_t *occ, int X, int Y,
                double ox, double oy) {
    std::unique_ptr<Front> f(new Front());
    if (poly_params) f->conf.poly_params = {poly_params[0], poly_params[1], poly_params[2]};
    f->conf.kernel_size = ks;
    f->conf.kernel_yaw_num = K;
    f->conf.occupancy_resolution = res;
    f->conf.front_end_safeh = safeh;
    Quiet q;
    f->shape.reset(make_shape(name ? name : "", f->conf));  // the constructor runs initShape
    if (!f->shape) return nullptr;
    f->grid = std::make_shared<GridMap3D>();
    GridMap3D &G = *f->grid;
    G.X_size = X; G.Y_size = Y; G.Z_size = 1; G.totalsize = X * Y;
    G.grid_resolution = res;
    G.boundary_xyzmin = Vector3d(ox, oy, 0.0);
    G.boundary_xyzmax = Vector3d(ox + X * res, oy + Y * res, res);
    G.grid_map_store.assign((size_t)X * Y, 0.0);
    for (size_t i = 0; i < (size_t)X * Y; ++i) G.grid_map_store[i] = occ[i] ? 1.0 : 0.0;
    G.grid_map = G.grid_map_store.data();
    f->env = std::make_shared<PCSmapManager>();
    f->env->boundary_xyzmin = G.boundary_xyzmin;
    f->env->boundary_xyzmax = G.boundary_xyzmax;
    f->env->occupancy_resolution = res;
    f->env->occupancy_map = f->grid;
    uint8_t *mk = f->env->generateMapKernel2D(ks);
    const int h = (ks - 1) / 2;
    f->mk_len = (X + 2 * h) * ((Y + 2 * h + 7) / 8);
    f->kernel_bytes.assign(mk, mk + f->mk_len);
    f->kernel_bytes.push_back(0);
    delete[] mk;
    f->env->mk = f->kernel_bytes.data();
    f->sv = std::make_shared<SweptVolumeManager>();
    SweptVolumeManager &S = *f->sv;
    S.map_kernel = f->kernel_bytes.data();
    S.map_Xsize = X; S.map_Ysize = Y; S.map_Zsize = 1;
    S.config = f->conf;
    S.kernel_count = K;    // sw_manager.hpp:241-242
    S.kernelsize = ks;
    S.current_robot_shape = f->shape.get();
    S.grid = f->grid.get();
    f->astar.initGridMap(f->env, f->sv);
    f->astar.kernel_size = ks;  // plan_manager.cpp:71
    return f.release();
}
void rf_destroy(void *h) { delete (Front *)h; }

// generateMapKernel2D's bytes ((X + 2h) rows of ceil((Y + 2h) / 8)); returns the length
int rf_map_kernel(void *h, uint8_t *out) {
    Front *f = (Front *)h;
    if (out) std::memcpy(out, f->kernel_bytes.data(), f->mk_len);
    return f->mk_len;
}
// initShape's kernels: yaw [K], cells [K][ks][ks], bytes [K][ks][(ks+7)/8]
void rf_kernels(void *h, double *yaw, uint8_t *cells, uint8_t *bytes) {
    Front *f = (Front *)h;
    const int ks = f->conf.kernel_size, K = f->conf.kernel_yaw_num, bl = (ks + 7) / 8;
    for (int k = 0; k < K; ++k) {
        yaw[k] = f->shape->shape_kernels[k].yaw;
        for (int a = 0; a < ks * ks; ++a) cells[(size_t)k * ks * ks + a] = f->shape->shape_kernels[k].map[a] ? 1 : 0;
        std::memcpy(bytes + (size_t)k * ks * bl, f->shape->byte_shape_kernels[k].map, (size_t)ks * bl);
    }
}
// kernelConv<byte>(k, (i, j, 0)) for n triples (k, i, j)
void rf_kernel_conv(void *h, int byte_variant, int64_t n, const int32_t *kij, uint8_t *out) {
    SweptVolumeManager &S = *((Front *)h)->sv;
    for (int64_t q = 0; q < n; ++q) {
        const Vector3i ind(kij[3 * q + 1], kij[3 * q + 2], 0);
        out[q] = byte_variant ? S.kernelConv<true>(kij[3 * q], ind) : S.kernelConv<false>(kij[3 * q], ind);
    }
}
// checkKernelValue(father_yaw, child_yaw, (i, j, 0)); child_yaw = father_yaw when it fails
void rf_check_kernel_value(void *h, int64_t n, const double *fy, const int32_t *ij, uint8_t *ok, double *cy) {
    SweptVolumeManager &S = *((Front *)h)->sv;
    for (int64_t q = 0; q < n; ++q) {
        double c = fy[q];
        ok[q] = S.checkKernelValue(fy[q], c, Vector3i(ij[2 * q], ij[2 * q + 1], 0)) ? 1 : 0;
        cy[q] = c;
    }
}
// getPointsInAABB2D(centre (cx, cy, 0), hbx, hby): writes up to cap points (x, y), returns how many there are
int64_t rf_points_in_aabb(void *h, double cx, double cy, double hbx, double hby, double *xy, int64_t cap) {
    std::vector<Eigen::Vector2d> pts;
    ((Front *)h)->env->getPointsInAABB2D(Vector3d(cx, cy, 0.0), hbx, hby, pts);
    for (int64_t i = 0; i < (int64_t)pts.size() && i < cap; ++i) { xy[2 * i] = pts[i](0); xy[2 * i + 1] = pts[i](1); }
    return (int64_t)pts.size();
}
// The A* node test for n nodes (cell node_ij, yaw node_yaw) and their 9 cells (di-major), [n][9] outputs:
//   ok: the cell is among the successors AstarGetSucc returns (run on the node with every neighbour unseen);
//   child_yaw: the yaw AstarGetSucc gives a successor; for the others, checkKernelValue's (the father's yaw when it fails);
//   parts: each condition on its own, from the same cut methods — bit 0 isIndexValid && !isIndexOccupiedFlate(0), bit 1
//          isIndexValid && checkKernelValue, bit 2 isIndexValid && checkSubSWCollision(state1, state2, getPointsInAABB2D of the
//          cell's centre, kernel_size/2+1), state2's yaw being checkKernelValue's.
void rf_expand(void *h, int64_t n, const int32_t *node_ij, const double *node_yaw, uint8_t *ok, double *child_yaw, uint8_t *parts) {
    Front *f = (Front *)h;
    GridMap3D &G = *f->grid;
    SweptVolumeManager &S = *f->sv;
    AstarPathSearcher &A = f->astar;
    const int hb = A.kernel_size / 2 + 1;
    for (int64_t q = 0; q < n; ++q) {
        const int ix = node_ij[2 * q], iy = node_ij[2 * q + 1];
        const double fy = node_yaw[q];
        for (int di = -1; di < 2; ++di)
            for (int dj = -1; dj < 2; ++dj)
                if (G.isIndexValid(ix + di, iy + dj, 0)) A.GridNodeMap[ix + di][iy + dj][0]->reset();
        GridNode *cur = A.GridNodeMap[ix][iy][0];
        cur->yaw = fy;
        vector<GridNode *> succ;
        vector<double> cost;
        A.AstarGetSucc(cur, succ, cost);
        for (int m = 0; m < 9; ++m) {
            const int di = m / 3 - 1, dj = m % 3 - 1;
            const Vector3i vi(ix + di, iy + dj, 0);
            const int64_t o = 9 * q + m;
            uint8_t p = 0;
            double cy = fy;
            if (G.isIndexValid(vi)) {
                if (!G.isIndexOccupiedFlate(vi, 0)) p |= 1;
                if (S.checkKernelValue(fy, cy, vi)) p |= 2;
                Vector3d s1 = G.getGridCubeCenter(Vector3i(ix, iy, 0));
                s1(2) = fy;
                Vector3d s2 = G.getGridCubeCenter(vi);
                s2(2) = 0;
                vector<Eigen::Vector2d> pts;
                f->env->getPointsInAABB2D(s2, hb, hb, pts);
                s2(2) = cy;
                if (S.checkSubSWCollision(s1, s2, pts)) p |= 4;
            }
            parts[o] = p;
            ok[o] = 0;
            child_yaw[o] = cy;
            for (GridNode *s : succ)
                if (s->index(0) == vi(0) && s->index(1) == vi(1)) { ok[o] = 1; child_yaw[o] = s->yaw; }
        }
    }
}
// AstarPathSearch + getPath for n start/goal pairs (z = 0): paths [n][max_path][3] (x, y, yaw), len (0: none, or longer than
// max_path), expansions (AstarGetSucc calls), found (success_flag)
void rf_astar(void *h, int n, const double *start_xy, const double *goal_xy, int max_path, double *paths, int32_t *len, int32_t *expansions,
              uint8_t *found) {
    AstarPathSearcher &A = ((Front *)h)->astar;
    for (int q = 0; q < n; ++q) {
        A.reset();
        A.success_flag = false;
        ros::time_default_constructions = 0;
        A.AstarPathSearch(Vector3d(start_xy[2 * q], start_xy[2 * q + 1], 0.0), Vector3d(goal_xy[2 * q], goal_xy[2 * q + 1], 0.0));
        expansions[q] = (int32_t)(ros::time_default_constructions / 3);
        found[q] = A.success_flag ? 1 : 0;
        len[q] = 0;
        if (A.success_flag) {
            vector<Vector3d> p = A.getPath();
            if ((int)p.size() <= max_path) {
                len[q] = (int32_t)p.size();
                for (size_t i = 0; i < p.size(); ++i)
                    for (int d = 0; d < 3; ++d) paths[((size_t)q * max_path + i) * 3 + d] = p[i](d);
            }
        }
    }
}

}  // extern "C"
