// oracle/ref_path_shim.cpp — TEST INFRASTRUCTURE: the REFERENCE'S OWN SOURCE of the hot path, compiled where it lies.
//
// Builds oracle/_ref/libref_path_<variant>.so (git-ignored; `make -C oracle ref_path`, only where /root/reference exists):
//   * `utils/trajectory.hpp` and `utils/minco.hpp` are #included WHOLE from /root/reference/src/utils/include;
//   * the shape classes (Shape.hpp), the SweptVolumeManager query methods (sw_manager.hpp) and the TrajOptimizer penalty
//     methods (back_end_optimizer.hpp) are #included from oracle/_ref/gen/*.inc, which oracle/ref_extract.py cuts VERBATIM
//     out of those files (they cannot be included whole: ROS / PCL / libigl / yaml members);
//   * Eigen is oracle/ref_shim/Eigen (a minimal stand-in, see its header for the one arithmetic degree of freedom and how
//     the tests neutralise it).
// What is OURS in this file is scaffolding only: the `Config` fields the code reads, a `BasicShape` base holding
// `trans/Rotate` (its constructor body is the verbatim fragment Shape.hpp:287-294), class shells around the verbatim
// methods with exactly the members they touch, and a C API (`ref_*`) mirroring oracle_capi.cpp's `orc_*` so that
// tests/test_oracle_ref_pin.py can run oracle and reference through the same calls and compare BITWISE.
//
// Variants (Makefile): glibc (the reference as it runs on x86-64: glibc libm, -O3, no FMA contraction) and portable
// (-DREF_LIBM_PORTABLE: every sin/cos/atan2 in the reference text is redirected to oracle/portable_sincos.hpp, the pinned
// fdlibm algorithm the CUDA kernels implement, so that reference == oracle == CUDA can be stated bit for bit).
#include <algorithm>
#include <cassert>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <functional>
#include <iostream>
#include <map>
#include <memory>
#include <set>
#include <sstream>
#include <string>
#include <vector>

#include <omp.h>

#ifdef REF_LIBM_PORTABLE
#include "portable_sincos.hpp"
namespace ref_libm {
inline double psin(double x) { double s, c; oracle::psc::sincos(x, s, c); return s; }
inline double pcos(double x) { double s, c; oracle::psc::sincos(x, s, c); return c; }
inline double patan2(double y, double x) { return oracle::psc::atan2(y, x); }
}  // namespace ref_libm
// both spellings the reference uses (`std::sin(x)` and `sin(x)`) must resolve after the textual redirection below
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
#include "pcl/stub.hpp"

#ifdef REF_LIBM_PORTABLE
// textual redirection of the libm calls in everything included from here on (reference text only)
#define sin psin
#define cos pcos
#define atan2 patan2
#endif

using namespace Eigen;  // utils/config.hpp:10
using namespace std;    // utils/config.hpp:11, Shape.hpp:33

// ---- utils/config.hpp:13-… : the fields the path reads ----------------------------------------------------------------
struct Config {
    int threads_num{12};
    vector<double> poly_params{0.0, 0.0, 0.0};
    int kernel_yaw_num{18};
    int kernel_size{17};
    double occupancy_resolution{1.0};
    double front_end_safeh{0.0};
    double safety_hor{0.7};
    double weight_p{60.0};
    string inputdata;
};

#include <utils/trajectory.hpp>  // WHOLE reference header (Piece<D>, Trajectory<D>)
#include <utils/minco.hpp>       // WHOLE reference header (BandedSystem, MINCO_S2NU/S3NU/S4NU)

#include "ref_shape_scaffold.inc"  // BasicShape scaffolding + the verbatim shape classes (Shape.hpp)

#include "_ref/gen/sw_macros.inc"     // TRAJ_ORDER, useScale, useNumer, pi (sw_manager.hpp:16-20)
#include "_ref/gen/sw_sampleset.inc"  // CircleCoord2D, SampleSet2D (sw_manager.hpp:25-124)

class SweptVolumeManager {
  public:
    double traj_duration{0.0};
    Config config;
    Trajectory<TRAJ_ORDER> traj;
    double momentum{0.0};
    double t_min{0.0};
    double t_max{1.0};
    BasicShape *current_robot_shape{nullptr};
#include "_ref/gen/sw_methods.inc"  // updateTraj … gradientDescent (sw_manager.hpp:374-1325, the methods on the path)
};

class TrajOptimizer {
  public:
    minco::MINCO_S3NU minco;
    SweptVolumeManager *sv_manager{nullptr};
    Trajectory<TRAJ_ORDER> step_traj;
    double rho{3.8};
    Config conf;
    double weight_p{60.0};
    double safety_hor{0.7};
    int threads_num{1};
    int parallel_points_num{0};
    std::vector<Eigen::Vector3d> parallel_points;
    double ori_cost_pos{0.0};
    int temporalDim{0}, spatialDim{0};
    Eigen::VectorXd times;
    Eigen::Matrix3Xd points;
    Eigen::MatrixX3d partialGradByCoeffs;
    Eigen::VectorXd partialGradByTimes;
    Eigen::Matrix3Xd gradByPoints;
    Eigen::VectorXd gradByTimes;
    double cost_pos{0}, cost_other{0}, cost_total{0};
#include "_ref/gen/opt_methods.inc"  // forwardT/P, backwardGradT/P, smoothedL1, costFunctionLmbmParallel, the penalty loop
};

#ifdef REF_LIBM_PORTABLE
#undef sin
#undef cos
#undef atan2
#endif
#undef pi

// =====================================================================================================================
// C API (ours): thin calls into the reference objects above
// =====================================================================================================================
namespace {
struct Quiet {  // the reference prints from constructors / initShape
    std::streambuf *old;
    std::ostringstream sink;
    Quiet() : old(std::cout.rdbuf(sink.rdbuf())) {}
    ~Quiet() { std::cout.rdbuf(old); }
};

BasicShape *make_shape(const char *name, const double *poly_params, const double *poly_xy, int poly_n, int ks, int K, double res,
                       double safeh) {
    Config conf;
    if (poly_params) conf.poly_params = {poly_params[0], poly_params[1], poly_params[2]};
    conf.kernel_size = ks;
    conf.kernel_yaw_num = K;
    conf.occupancy_resolution = res;
    conf.front_end_safeh = safeh;
    std::string n = name ? name : "";
    Quiet q;
    // registry of sw_manager.hpp:187-235 (the lambdas only `new` the class); unknown names fall back to the rectangle
    // Polygon of sw_manager.hpp:363-372
    if (poly_xy && poly_n > 0) {
        Eigen::MatrixX2d v(poly_n, 2);
        for (int i = 0; i < poly_n; ++i) v.row(i) = Eigen::Vector2d(poly_xy[2 * i], poly_xy[2 * i + 1]);
        return new Polygon(conf, v);
    }
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

struct RefCtx {
    TrajOptimizer opt;
    SweptVolumeManager sv;
    Eigen::Matrix3d init_s, final_s;
    int N = 0;
    ~RefCtx() { delete sv.current_robot_shape; }
};

// MINCO b (6N x 3 column-major) -> Trajectory<5>: the expression of MINCO_S3NU::getTrajectory (minco.hpp:515-528)
void traj_from_coeffs(int N, const double *T, const double *coeffs, Trajectory<5> &traj) {
    Eigen::MatrixX3d b(6 * N, 3);
    for (int d = 0; d < 3; ++d)
        for (int r = 0; r < 6 * N; ++r) b(r, d) = coeffs[d * 6 * N + r];
    traj.clear();
    traj.reserve(N);
    for (int i = 0; i < N; i++) traj.emplace_back(T[i], b.block<6, 3>(6 * i, 0).transpose().rowwise().reverse());
}
}  // namespace

extern "C" {

const char *ref_variant() {
#ifdef REF_LIBM_PORTABLE
    return "portable";
#else
    return "glibc";
#endif
}
int ref_redux_order() { return REF_SHIM_REDUX; }

// BasicShape::getonlySDF / getonlyGrad1 over n body-frame points (stride 3)
void ref_shape_sdf(const char *name, const double *poly_params, const double *poly_xy, int poly_n, int64_t n, const double *rel,
                   double *out) {
    std::unique_ptr<BasicShape> S(make_shape(name, poly_params, poly_xy, poly_n, 3, 2, 1.0, 0.0));
    for (int64_t i = 0; i < n; ++i) out[i] = S->getonlySDF(Eigen::RowVector3d(rel[3 * i], rel[3 * i + 1], rel[3 * i + 2]));
}
void ref_shape_grad1(const char *name, const double *poly_params, const double *poly_xy, int poly_n, int64_t n, const double *rel,
                     double *out3) {
    std::unique_ptr<BasicShape> S(make_shape(name, poly_params, poly_xy, poly_n, 3, 2, 1.0, 0.0));
    for (int64_t i = 0; i < n; ++i) {
        Eigen::Vector3d g = S->getonlyGrad1(Eigen::RowVector3d(rel[3 * i], rel[3 * i + 1], rel[3 * i + 2]));
        out3[3 * i] = g(0); out3[3 * i + 1] = g(1); out3[3 * i + 2] = g(2);
    }
}
// BasicShape::initShape (Shape.hpp:384-430): yaw-indexed occupancy kernels; cells [K][ks][ks], bytes [K][ks][(ks+7)/8]
void ref_shape_kernels(const char *name, const double *poly_params, int ks, int K, double res, double safeh, double *yaw_out,
                       uint8_t *cells_out, uint8_t *bytes_out) {
    std::unique_ptr<BasicShape> S(make_shape(name, poly_params, nullptr, 0, ks, K, res, safeh));  // ctor runs initShape
    int bl = (ks + 7) / 8;
    for (int k = 0; k < K; ++k) {
        yaw_out[k] = S->shape_kernels[k].yaw;
        for (int a = 0; a < ks; ++a)
            for (int b = 0; b < ks; ++b) cells_out[((size_t)k * ks + a) * ks + b] = S->shape_kernels[k].map[a * ks + b] ? 1 : 0;
        std::memcpy(bytes_out + (size_t)k * ks * bl, S->byte_shape_kernels[k].map, (size_t)ks * bl);
    }
}

void ref_smoothed_l1(int64_t n, const double *x, double mu, double *f, double *df, uint8_t *ret) {
    for (int64_t i = 0; i < n; ++i) {
        double ff = 0, dd = 0;
        ret[i] = TrajOptimizer::smoothedL1(x[i], mu, ff, dd) ? 1 : 0;
        f[i] = ff; df[i] = dd;
    }
}

void *ref_create(const char *name, const double *poly_params, const double *poly_xy, int poly_n, double weight_p, double safety_hor,
                 double rho, int threads) {
    RefCtx *c = new RefCtx();
    c->sv.current_robot_shape = make_shape(name, poly_params, poly_xy, poly_n, 3, 2, 1.0, 0.0);
    c->opt.sv_manager = &c->sv;
    c->opt.weight_p = weight_p;
    c->opt.safety_hor = safety_hor;
    c->opt.rho = rho;
    c->opt.threads_num = threads > 0 ? threads : 1;
    return c;
}
void ref_destroy(void *h) { delete (RefCtx *)h; }
void ref_set_threads(void *h, int n) { ((RefCtx *)h)->opt.threads_num = n > 0 ? n : 1; }

void ref_set_points(void *h, const double *pts, int64_t P, int stride) {
    RefCtx *c = (RefCtx *)h;
    c->opt.parallel_points.resize((size_t)P);
    for (int64_t k = 0; k < P; ++k)
        c->opt.parallel_points[(size_t)k] = Eigen::Vector3d(pts[k * stride], pts[k * stride + 1], stride > 2 ? pts[k * stride + 2] : 0.0);
    c->opt.parallel_points_num = (int)P;
}
void ref_set_traj(void *h, int N, const double *T, const double *coeffs) {
    RefCtx *c = (RefCtx *)h;
    c->N = N;
    traj_from_coeffs(N, T, coeffs, c->opt.step_traj);
    c->sv.updateTraj(c->opt.step_traj);
}
double ref_traj_duration(void *h) { return ((RefCtx *)h)->sv.traj_duration; }
void ref_traj_pos(void *h, double t, double *out) { Eigen::Vector3d p = ((RefCtx *)h)->sv.traj.getPos(t); out[0] = p(0); out[1] = p(1); out[2] = p(2); }
void ref_traj_vel(void *h, double t, double *out) { Eigen::Vector3d p = ((RefCtx *)h)->sv.traj.getVel(t); out[0] = p(0); out[1] = p(1); out[2] = p(2); }
int ref_locate_piece(void *h, double t, double *t_local) { int i = ((RefCtx *)h)->sv.traj.locatePieceIdx(t); *t_local = t; return i; }
double ref_sdf_at(void *h, const double *p, double t) { return ((RefCtx *)h)->sv.getSDFAtTimeStamp<false>(Eigen::Vector3d(p[0], p[1], p[2]), t); }
double ref_sdf_dot_at(void *h, const double *p, double t) { return ((RefCtx *)h)->sv.getSDF_DOTAtTimeStamp<false>(Eigen::Vector3d(p[0], p[1], p[2]), t); }
double ref_choice_t_init(void *h, const double *p, double dt) { return ((RefCtx *)h)->sv.choiceTInit<false>(Eigen::Vector3d(p[0], p[1], p[2]), dt); }
void ref_gradient_descent(void *h, const double *p, double tmin, double tmax, double x0, double *fx, double *x) {
    ((RefCtx *)h)->sv.gradientDescent(0.0, tmin, tmax, x0, *fx, *x, Eigen::Vector3d(p[0], p[1], p[2]));
}
// getSDFofSweptVolume<false,true> per point (stride 3): sdf, t*, body-frame FD gradient
void ref_query_outer(void *h, int64_t n, const double *pts, double *sdf, double *tstar, double *g3) {
    RefCtx *c = (RefCtx *)h;
#pragma omp parallel for num_threads(c->opt.threads_num) schedule(dynamic)
    for (int64_t k = 0; k < n; ++k) {
        Eigen::Vector3d g = Eigen::Vector3d::Zero();
        double ts = 0.0;
        sdf[k] = c->sv.getSDFofSweptVolume<false, true>(Eigen::Vector3d(pts[3 * k], pts[3 * k + 1], pts[3 * k + 2]), ts, g);
        tstar[k] = ts;
        g3[3 * k] = g(0); g3[3 * k + 1] = g(1); g3[3 * k + 2] = g(2);
    }
}
// getTrueSDFofSweptVolume<true> per point: for sdf <= 0 the gradient is the WORLD-frame unit vector of the GSIP branch
void ref_query(void *h, int64_t n, const double *pts, double *sdf, double *tstar, double *g3) {
    RefCtx *c = (RefCtx *)h;
#pragma omp parallel for num_threads(c->opt.threads_num) schedule(dynamic)
    for (int64_t k = 0; k < n; ++k) {
        Eigen::Vector3d g = Eigen::Vector3d::Zero();
        double ts = 0.0;
        sdf[k] = c->sv.getTrueSDFofSweptVolume<true>(Eigen::Vector3d(pts[3 * k], pts[3 * k + 1], pts[3 * k + 2]), ts, g, false);
        tstar[k] = ts;
        g3[3 * k] = g(0); g3[3 * k + 1] = g(1); g3[3 * k + 2] = g(2);
    }
}
// addSaftyPenaOnSweptVolumeParallelTrueSDF (accumulating): coeffs / gradC 6N x 3 column-major
void ref_cost_grad(void *h, int N, const double *T, const double *coeffs, double *cost_io, double *gradT_io, double *gradC_io) {
    RefCtx *c = (RefCtx *)h;
    ref_set_traj(h, N, T, coeffs);
    Eigen::VectorXd Tv(N), gT(N);
    Eigen::MatrixX3d b(6 * N, 3), gC(6 * N, 3);
    for (int i = 0; i < N; ++i) { Tv(i) = T[i]; gT(i) = gradT_io[i]; }
    for (int d = 0; d < 3; ++d)
        for (int r = 0; r < 6 * N; ++r) { b(r, d) = coeffs[d * 6 * N + r]; gC(r, d) = gradC_io[d * 6 * N + r]; }
    double cost = *cost_io;
    TrajOptimizer::addSaftyPenaOnSweptVolumeParallelTrueSDF(&c->opt, Tv, b, cost, gT, gC);
    *cost_io = cost;
    for (int i = 0; i < N; ++i) gradT_io[i] = gT(i);
    for (int d = 0; d < 3; ++d)
        for (int r = 0; r < 6 * N; ++r) gradC_io[d * 6 * N + r] = gC(r, d);
}

// ---- MINCO_S3NU (whole reference class) --------------------------------------------------------------------------------
// init_s / final_s: 3x3 column-major (columns pos, vel, acc) as plan_manager.cpp:143-147 builds them
void ref_set_conditions(void *h, const double *init_s, const double *final_s, int N) {
    RefCtx *c = (RefCtx *)h;
    for (int j = 0; j < 3; ++j)
        for (int i = 0; i < 3; ++i) { c->init_s(i, j) = init_s[j * 3 + i]; c->final_s(i, j) = final_s[j * 3 + i]; }
    c->N = N;
    c->opt.temporalDim = N;           // back_end_optimizer.cpp:13-19
    c->opt.spatialDim = 3 * (N - 1);
    c->opt.minco.setConditions(c->init_s, c->final_s, N);
}
// costFunctionLmbmParallel(ptr, x, g, n) verbatim
double ref_evaluate(void *h, const double *x, double *g, int n) { return TrajOptimizer::costFunctionLmbmParallel(&((RefCtx *)h)->opt, x, g, n); }
void ref_last_costs(void *h, double *out3) { RefCtx *c = (RefCtx *)h; out3[0] = c->opt.cost_pos; out3[1] = c->opt.cost_other; out3[2] = c->opt.cost_total; }
// forward: q (3 x (N-1) column-major), T -> b (6N x 3 column-major), energy, dE/dc, dE/dT
void ref_minco_forward(void *h, const double *q, const double *T, double *b_out, double *energy, double *gdC_out, double *gdT_out) {
    RefCtx *c = (RefCtx *)h;
    int N = c->N;
    Eigen::Matrix3Xd P(3, N - 1);
    Eigen::VectorXd Tv(N);
    for (int i = 0; i < N - 1; ++i) for (int d = 0; d < 3; ++d) P(d, i) = q[3 * i + d];
    for (int i = 0; i < N; ++i) Tv(i) = T[i];
    c->opt.minco.setParameters(P, Tv);
    const Eigen::MatrixX3d &b = c->opt.minco.getCoeffs();
    Eigen::MatrixX3d gdC;
    Eigen::VectorXd gdT;
    c->opt.minco.getEnergy(*energy);
    c->opt.minco.getEnergyPartialGradByCoeffs(gdC);
    c->opt.minco.getEnergyPartialGradByTimes(gdT);
    for (int d = 0; d < 3; ++d)
        for (int r = 0; r < 6 * N; ++r) { b_out[d * 6 * N + r] = b(r, d); gdC_out[d * 6 * N + r] = gdC(r, d); }
    for (int i = 0; i < N; ++i) gdT_out[i] = gdT(i);
}
// adjoint: (dJ/dc, dJ/dT) -> (dJ/dq 3 x (N-1) column-major, dJ/dT)
void ref_minco_propagate(void *h, const double *gdC, const double *gdT, double *gradP_out, double *gradT_out) {
    RefCtx *c = (RefCtx *)h;
    int N = c->N;
    Eigen::MatrixX3d pc(6 * N, 3);
    Eigen::VectorXd pt(N), gt;
    Eigen::Matrix3Xd gp;
    for (int d = 0; d < 3; ++d) for (int r = 0; r < 6 * N; ++r) pc(r, d) = gdC[d * 6 * N + r];
    for (int i = 0; i < N; ++i) pt(i) = gdT[i];
    c->opt.minco.propogateGrad(pc, pt, gp, gt);
    for (int i = 0; i < N - 1; ++i) for (int d = 0; d < 3; ++d) gradP_out[3 * i + d] = gp(d, i);
    for (int i = 0; i < N; ++i) gradT_out[i] = gt(i);
}
// tau <-> T maps (back_end_optimizer.hpp:199-289)
void ref_forward_T(int n, const double *tau, double *T) { Eigen::VectorXd Tv; TrajOptimizer::forwardT(tau, Tv, n); for (int i = 0; i < n; ++i) T[i] = Tv(i); }
void ref_backward_T(int n, const double *T, double *tau) { Eigen::VectorXd Tv(n), tv; for (int i = 0; i < n; ++i) Tv(i) = T[i]; TrajOptimizer::backwardT(Tv, tv); for (int i = 0; i < n; ++i) tau[i] = tv(i); }

}  // extern "C"
