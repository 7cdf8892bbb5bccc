// oracle/ref_mid_shim.cpp — TEST INFRASTRUCTURE: the REFERENCE'S OWN SOURCE of the mid end, compiled where it lies.
//
// Builds oracle/_ref/libref_mid.so (git-ignored; `make -C oracle ref_path`, only where /root/reference exists):
//   * `utils/minco.hpp`, `utils/trajectory.hpp`, `utils/flatness.hpp` and `utils/lbfgs.hpp` (the reference's patched L-BFGS) are
//     #included WHOLE from /root/reference/src/utils/include;
//   * OriTraj's member functions (planner_algorithm/mid_end.hpp: the tau / xi maps, smoothedL1, grad_cost_dir, addPosePenalty,
//     costFunction, costaltitude, gradaltitude, WC2, addTimeIntPenalty, earlyExit) and OriTraj::getOriTraj (src/mid_end.cpp) come
//     from oracle/_ref/gen/mid_*.inc, cut VERBATIM by oracle/ref_extract.py (the header cannot be included whole: ROS members);
//   * Eigen is the stand-in oracle/ref_shim/Eigen.
// OURS: the class shell with the members those functions touch, empty ROS / debug stubs, and the C API below
// (tests/test_oracle_mid.py compares the product's host/mid_end.hpp with it).
#include <algorithm>
#include <cassert>
#include <chrono>
#include <cmath>
#include <cstring>
#include <iostream>
#include <memory>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

#include <Eigen/Eigen>

using namespace Eigen;
using namespace std;

// ---- stubs for what the verbatim text mentions besides arithmetic -----------------------------------------------------------------
namespace ros {
struct Time { static Time now() { return Time(); } };
struct NodeHandle {};
struct Publisher {};
}  // namespace ros
namespace debug_publisher {
inline void DBSendNew(const std::string &, const std::string &) {}
}  // namespace debug_publisher
#define ROS_WARN_STREAM(x) do { } while (0)

#include "utils/trajectory.hpp"
#include "utils/minco.hpp"
#include "utils/flatness.hpp"
#include "utils/lbfgs.hpp"

#define TRAJ_ORDER 5  // mid_end.hpp:14

struct Config {  // utils/config.hpp: the fields the mid end reads
    int mem_size{16};
    int past{64};
    double min_step{1.0e-32};
    double g_epsilon{0.0};
    double relCostTolMidEnd{1.0e-10};
    bool enableearlyExit{false};
    int debugpause{0};
};

class OriTraj {
   public:
    minco::MINCO_S3NU minco;
    flatness::FlatnessMap flatmap;
    Trajectory<TRAJ_ORDER> step_traj;
    double rho, vmax, omgmax, weight_v, weight_omg;
    int integralRes;
    Eigen::Matrix3d initState, finalState;
    Eigen::Matrix3Xd accelerations, ref_points;
    std::vector<Eigen::Matrix3d> att_constraints;
    Eigen::Matrix3Xd points;
    Eigen::VectorXd times;
    Eigen::Matrix3Xd gradByPoints;
    Eigen::VectorXd gradByTimes;
    Eigen::MatrixX3d partialGradByCoeffs;
    Eigen::VectorXd partialGradByTimes;
    int pieceN, spatialDim, temporalDim;
    double smooth_fac;
    Config conf;
    double weightPR, weightAR;
    int iter = 0;
    void drawDebugTraj() {}
#include "_ref/gen/mid_methods.inc"
    bool getOriTraj(const Eigen::Matrix3d initS, const Eigen::Matrix3d finalS, const std::vector<Eigen::Vector3d> &Q, Eigen::VectorXd T,
                    std::vector<Eigen::Vector3d> acc_list, std::vector<Eigen::Matrix3d> rot_list, const int N, Trajectory<TRAJ_ORDER> &traj,
                    Eigen::VectorXd &opt_x);
};
#include "_ref/gen/mid_getoritraj.inc"

// ---- C API ---------------------------------------------------------------------------------------------------------------------------
namespace {
struct MidCfg {  // == svsdf_mid_config (include/svsdf.h)
    double rho_mid_end, vmax, omgmax, weight_v, weight_omg, weight_pr, weight_ar, smoothingEps;
    int integralIntervs;
    double vehicleMass, gravAcc, horizDrag, vertDrag, parasDrag, speedEps;
    int mem_size, past;
    double min_step, g_epsilon, relCostTolMidEnd;
    int max_iterations, cancel_after, solver;
};
void configure(OriTraj &o, const MidCfg &c) {  // OriTraj::setParam (mid_end.hpp:333-359) without the ROS lines
    o.weightPR = c.weight_pr; o.weightAR = c.weight_ar; o.rho = c.rho_mid_end; o.vmax = c.vmax; o.omgmax = c.omgmax;
    o.weight_v = c.weight_v; o.weight_omg = c.weight_omg; o.smooth_fac = c.smoothingEps; o.integralRes = c.integralIntervs;
    o.flatmap.reset(c.vehicleMass, c.gravAcc, c.horizDrag, c.vertDrag, c.parasDrag, c.speedEps);
    o.conf.mem_size = c.mem_size; o.conf.past = c.past; o.conf.min_step = c.min_step; o.conf.g_epsilon = c.g_epsilon;
    o.conf.relCostTolMidEnd = c.relCostTolMidEnd;
}
Matrix3d mat3(const double *p) { Matrix3d m; for (int c = 0; c < 3; ++c) for (int r = 0; r < 3; ++r) m(r, c) = p[3 * c + r]; return m; }
struct Quiet {  // the reference prints every iteration
    std::streambuf *old;
    std::ostringstream sink;
    Quiet() : old(std::cout.rdbuf(sink.rdbuf())) {}
    ~Quiet() { std::cout.rdbuf(old); }
};
}  // namespace

extern "C" {
// the state getOriTraj sets up before it calls the solver (mid_end.cpp:14-43), then one costFunction call at x
int ref_mid_cost(const MidCfg *cfg, int N, const double *initS, const double *finalS, const double *Q, const double *rot_list, const double *x,
                 double *cost_out, double *grad_out) {
    OriTraj o;
    configure(o, *cfg);
    o.pieceN = N; o.temporalDim = N; o.spatialDim = 3 * (N - 1);
    o.initState = mat3(initS); o.finalState = mat3(finalS);
    o.minco.setConditions(o.initState, o.finalState, o.pieceN);
    o.ref_points.resize(3, N - 1); o.accelerations.resize(3, N - 1); o.att_constraints.clear();
    for (int i = 0; i < N - 1; ++i) {
        o.ref_points.col(i) = Vector3d(Q[3 * i], Q[3 * i + 1], Q[3 * i + 2]);
        o.accelerations.col(i) = Vector3d(0, 0, 1);
        o.att_constraints.push_back(mat3(rot_list + 9 * i));
    }
    o.gradByPoints.resize(3, N - 1); o.gradByPoints.setZero();
    const int n = N + 3 * (N - 1);
    VectorXd xv(n), g(n);
    for (int i = 0; i < n; ++i) xv(i) = x[i];
    double p_cost = 0.0;
    *cost_out = OriTraj::costFunction(&o, xv, g, p_cost);
    for (int i = 0; i < n; ++i) grad_out[i] = g(i);
    return 0;
}
// OriTraj::getOriTraj with the reference's own (patched) L-BFGS
int ref_mid_get_ori_traj(const MidCfg *cfg, int N, const double *initS, const double *finalS, const double *Q, const double *T_init,
                         const double *rot_list, double *opt_x_out, double *T_out, double *coeffs_out, int *iterations_out) {
    OriTraj o;
    configure(o, *cfg);
    std::vector<Vector3d> Qv, acc;
    std::vector<Matrix3d> rot;
    for (int i = 0; i < N - 1; ++i) {
        Qv.push_back(Vector3d(Q[3 * i], Q[3 * i + 1], Q[3 * i + 2]));
        acc.push_back(Vector3d(0, 0, 1));
        rot.push_back(mat3(rot_list + 9 * i));
    }
    VectorXd T(N);
    for (int i = 0; i < N; ++i) T(i) = T_init[i];
    Trajectory<TRAJ_ORDER> traj;
    VectorXd opt_x(N + 3 * (N - 1));
    opt_x.setZero();
    bool ok;
    {
        Quiet q;
        ok = o.getOriTraj(mat3(initS), mat3(finalS), Qv, T, acc, rot, N, traj, opt_x);
    }
    if (ok) for (int i = 0; i < N + 3 * (N - 1); ++i) opt_x_out[i] = opt_x(i);
    for (int i = 0; i < N; ++i) T_out[i] = o.times(i);
    const Eigen::MatrixX3d &b = o.minco.getCoeffs();
    for (int d = 0; d < 3; ++d)
        for (int r = 0; r < 6 * N; ++r) coeffs_out[d * 6 * N + r] = b(r, d);
    if (iterations_out) *iterations_out = o.iter;
    return ok ? 1 : 0;
}
}
