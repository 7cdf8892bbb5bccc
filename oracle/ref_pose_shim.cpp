// oracle/ref_pose_shim.cpp — TEST INFRASTRUCTURE: the REFERENCE'S OWN SOURCE of the pose-sampled obstacle penalty, compiled where it
// lies.
//
// Builds oracle/_ref/libref_pose_<variant>.so (git-ignored; `make -C oracle ref`, only where the reference tree exists):
//   * the shape classes: oracle/ref_shape_scaffold.inc over the fragments of oracle/ref_extract.py, as in libref_path_*;
//   * GridMap3D's members and PCSmapManager::projInMap: the fragments of oracle/ref_extract_front.py, as in libref_front_*;
//   * TrajOptimizer::smoothedL1 / grad_cost_p, SweptVolumeManager::posEva2Rel / getSDFWithGradWhenRobotAtState and
//     PCSmapManager::getPointsInAABB: oracle/_ref/pose/gen/*.inc, cut VERBATIM by oracle/ref_extract_pose.py;
//   * ros::Time: oracle/ref_shim/ros/time_stub.hpp (grad_cost_p only times itself with it).
// What is OURS is storage only (the members the cut methods read) and the C API at the bottom.  Choices:
//   * The map is the product's: X x Y x Z voxels of size res from lo, boundary_xyzmax = lo + (X, Y, Z) res (the map given as kernel
//     bytes has no cloud maximum), occupancy stored in GridMap3D's own layout (toAddr).
//   * bdx, bdy, bdz = 2 half (grad_cost_p reads bdx / 2: exact).
//   * `rotate` (back_end_optimizer.hpp:439) is declared uninitialised in addTimeIntPenalty; grad_cost_p sets five entries.  The caller
//     here passes it zero-initialised, as the product takes it.
// Variants (oracle/Makefile): glibc (the reference as it runs on x86-64) and portable (-DREF_LIBM_PORTABLE: the pinned fdlibm sin / cos the
// CUDA kernels implement).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <map>
#include <memory>
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

// `grad_yaw += -grad_out * gradp_rel.transpose() * (...)` (back_end_optimizer.hpp:1024) adds a 1 x 1 product to a double.  Eigen
// converts the 1 x 1 expression to its scalar; the stand-in has that conversion for assignment but not for the built-in +=, so it is
// spelled out here: the product's one coefficient, then the addition.
namespace Eigen {
inline double &operator+=(double &a, const Matrix<double, 1, 1> &b) { return a += static_cast<double>(b); }
}  // namespace Eigen

#ifdef REF_LIBM_PORTABLE
#define sin psin
#define cos pcos
#define atan2 patan2
#endif

using namespace Eigen;  // utils/config.hpp:10
using namespace std;    // utils/config.hpp:11

struct Config {  // utils/config.hpp: the fields the shapes read
    vector<double> poly_params{0.0, 0.0, 0.0};
    int kernel_yaw_num{18};
    int kernel_size{17};
    double occupancy_resolution{1.0};
    double front_end_safeh{0.0};
};

#include "ref_shape_scaffold.inc"  // BasicShape + the shape classes (Shape.hpp), as in libref_path_*
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
#include "_ref/pose/gen/pcs_pose_methods.inc"
    Vector3d boundary_xyzmin, boundary_xyzmax;
    double occupancy_resolution{1.0};
    GridMap3D::Ptr occupancy_map;
    uint8_t *mk{nullptr};
    typedef shared_ptr<PCSmapManager> Ptr;
};

class SweptVolumeManager {  // storage of sw_manager.hpp:129-153
  public:
    BasicShape *current_robot_shape{nullptr};
#include "_ref/pose/gen/sw_pose_methods.inc"
    typedef shared_ptr<SweptVolumeManager> Ptr;
};

class TrajOptimizer {  // storage of back_end_optimizer.hpp's TrajOptimizer: the members grad_cost_p reads
  public:
    SweptVolumeManager::Ptr sv_manager;
    PCSmapManager::Ptr pcsmap_manager;
    double safety_hor{0.7};
    double bdx{17.0}, bdy{17.0}, bdz{17.0};
    double total_AABB_time{0.0}, total_sdf_time{0.0};
#include "_ref/pose/gen/opt_pose_methods.inc"
};

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
struct Quiet {  // the shapes print from their constructors
    std::streambuf *old;
    std::ostringstream sink;
    Quiet() : old(std::cout.rdbuf(sink.rdbuf())) {}
    ~Quiet() { std::cout.rdbuf(old); }
};

BasicShape *make_shape(const char *name, const double *poly_params, const double *poly_xy, int poly_n) {
    Config conf;
    if (poly_params) conf.poly_params = {poly_params[0], poly_params[1], poly_params[2]};
    conf.kernel_size = 3;
    conf.kernel_yaw_num = 2;
    std::string n = name ? name : "";
    Quiet q;
    if (poly_xy && poly_n > 0) {
        Eigen::MatrixX2d v(poly_n, 2);
        for (int i = 0; i < poly_n; ++i) v.row(i) = Eigen::Vector2d(poly_xy[2 * i], poly_xy[2 * i + 1]);
        return new Polygon(conf, v);
    }
    // registry of sw_manager.hpp:187-235; unknown names fall back to the rectangle Polygon of sw_manager.hpp:363-372
#define REF_SHAPE(N) if (n == #N) return new N(conf);
    REF_SHAPE(sdUnevenCapsule) REF_SHAPE(sdCutDisk) REF_SHAPE(sdTrapezoid) REF_SHAPE(sdRhombus) REF_SHAPE(star)
    REF_SHAPE(sdTunnel) REF_SHAPE(sdHorseshoe) REF_SHAPE(sdHeart) REF_SHAPE(sdOrientedVesica) REF_SHAPE(sdRoundedCross)
    REF_SHAPE(sdRoundedX) REF_SHAPE(bigX) REF_SHAPE(sdMoon) REF_SHAPE(sdPie) REF_SHAPE(sdPie2) REF_SHAPE(sdArc)
    REF_SHAPE(Circle)
#undef REF_SHAPE
    Eigen::MatrixX2d rect(4, 2);
    rect.row(0) = Eigen::Vector2d(6, -0.1);
    rect.row(1) = Eigen::Vector2d(6, 0.1);
    rect.row(2) = Eigen::Vector2d(-6, 0.1);
    rect.row(3) = Eigen::Vector2d(-6, -0.1);
    return new Polygon(conf, rect);
}
}  // namespace

extern "C" {

const char *rp_variant() {
#ifdef REF_LIBM_PORTABLE
    return "portable";
#else
    return "glibc";
#endif
}

// grad_cost_p at n poses (x, y, yaw) against the map occ [X][Y][Z] (0 / 1, C order) at lo with voxel edge res, box half sizes half[3]
// and safety_hor: out[n][4] = (costp, gradp(0), gradp(1), grad_yaw).
void rp_grad_cost_p(const char *name, const double *poly_params, const double *poly_xy, int poly_n, const uint8_t *occ, int X, int Y,
                    int Z, const double *lo, double res, const double *half, double safety_hor, int64_t n, const double *poses,
                    double *out) {
    std::unique_ptr<BasicShape> shape(make_shape(name, poly_params, poly_xy, poly_n));
    auto grid = std::make_shared<GridMap3D>();
    GridMap3D &G = *grid;
    G.X_size = X; G.Y_size = Y; G.Z_size = Z; G.totalsize = X * Y * Z;
    G.grid_resolution = res;
    G.boundary_xyzmin = Vector3d(lo[0], lo[1], lo[2]);
    G.boundary_xyzmax = Vector3d(lo[0] + X * res, lo[1] + Y * res, lo[2] + Z * res);
    G.grid_map_store.assign((size_t)X * Y * Z, 0.0);
    for (int x = 0; x < X; ++x)
        for (int y = 0; y < Y; ++y)
            for (int z = 0; z < Z; ++z)
                G.grid_map_store[G.toAddr(x, y, z)] = occ[((size_t)x * Y + y) * Z + z] ? 1.0 : 0.0;
    G.grid_map = G.grid_map_store.data();
    TrajOptimizer opt;
    opt.pcsmap_manager = std::make_shared<PCSmapManager>();
    opt.pcsmap_manager->boundary_xyzmin = G.boundary_xyzmin;
    opt.pcsmap_manager->boundary_xyzmax = G.boundary_xyzmax;
    opt.pcsmap_manager->occupancy_resolution = res;
    opt.pcsmap_manager->occupancy_map = grid;
    opt.sv_manager = std::make_shared<SweptVolumeManager>();
    opt.sv_manager->current_robot_shape = shape.get();
    opt.safety_hor = safety_hor;
    opt.bdx = 2.0 * half[0];
    opt.bdy = 2.0 * half[1];
    opt.bdz = 2.0 * half[2];
    const Eigen::Matrix3d St = Eigen::Matrix3d::Identity();  // passed and never read (:484)
    const Eigen::Vector4d quat = Eigen::Vector4d::Zero();   // passed and never read
    for (int64_t k = 0; k < n; ++k) {
        Eigen::Matrix3d rotate = Eigen::Matrix3d::Zero();
        Eigen::Vector3d gradp;
        double grad_yaw = 0.0, costp = 0.0;
        opt.grad_cost_p(Eigen::Vector3d(poses[3 * k], poses[3 * k + 1], poses[3 * k + 2]), rotate, St, quat, gradp, grad_yaw, costp);
        out[4 * k] = costp;
        out[4 * k + 1] = gradp(0);
        out[4 * k + 2] = gradp(1);
        out[4 * k + 3] = grad_yaw;
    }
}

}  // extern "C"
