// oracle/oracle_capi.cpp — TEST INFRASTRUCTURE ONLY: C entry points (for ctypes) over the CPU oracle.
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs load this.
#include <omp.h>

#include <chrono>
#include <cstdio>
#include <cstring>

#include "frontend_oracle.hpp"
#include "minco_oracle.hpp"

using namespace oracle;

namespace {
Shape make_shape(const char *name, const double *poly_params, const double *poly_xy, int poly_n) {
    Shape S;
    S.id = shape_id_from_name(name ? name : "");
    if (poly_params) S.set_poly_params(poly_params[0], poly_params[1], poly_params[2]);
    if (S.id == SH_POLYGON) {
        if (poly_xy && poly_n >= 3) S.set_polygon(poly_xy, poly_n);
        else S.set_default_rect();
    }
    return S;
}
}  // namespace

extern "C" {

int orc_shape_id(const char *name) { return shape_id_from_name(name ? name : ""); }

// BasicShape::getonlySDF over n body-frame points (stride 3)
void orc_shape_sdf(const char *name, const double *poly_params, const double *poly_xy, int poly_n, int64_t n,
                   const double *rel, double *out) {
    Shape S = make_shape(name, poly_params, poly_xy, poly_n);
    for (int64_t i = 0; i < n; ++i) out[i] = shape_sdf(S, rel[3 * i], rel[3 * i + 1], rel[3 * i + 2]);
}
// BasicShape::getonlyGrad1
void orc_shape_grad1(const char *name, const double *poly_params, const double *poly_xy, int poly_n, int64_t n,
                     const double *rel, double *out3) {
    Shape S = make_shape(name, poly_params, poly_xy, poly_n);
    for (int64_t i = 0; i < n; ++i) shape_grad1(S, rel[3 * i], rel[3 * i + 1], rel[3 * i + 2], out3 + 3 * i);
}

// the oracle's sin/cos (portable fdlibm restatement, or glibc in the "glibc"/"fma" variants)
void orc_sincos(int64_t n, const double *x, double *s, double *c) {
    for (int64_t i = 0; i < n; ++i) psc::sincos(x[i], s[i], c[i]);
}

void orc_atan2(int64_t n, const double *y, const double *x, double *out) {
    for (int64_t i = 0; i < n; ++i) out[i] = psc::atan2(y[i], x[i]);
}

// atan2f: the pinned fdlibm code the winding-number traversal uses (host and device) beside the C library's
void orc_atan2f_pair(int64_t n, const float *y, const float *x, float *out_portable, float *out_libm) {
    for (int64_t i = 0; i < n; ++i) {
        out_portable[i] = svsdf::host::FwnBvh::atan2f_portable(y[i], x[i]);
        out_libm[i] = ::atan2f(y[i], x[i]);
    }
}

// ---- triangle-mesh functor (BasicShape::getonlySDF_igl, Shape.hpp:332-340); V: nv x 3 row-major, F: nf x 3 ----
static Shape make_mesh_shape(const double *poly_params, const double *V, int nv, const int *F, int nf) {
    Shape S;
    S.id = SH_MESH;
    if (poly_params) S.set_poly_params(poly_params[0], poly_params[1], poly_params[2]);
    S.set_mesh(V, nv, F, nf);
    return S;
}
// what: 0 sdf, 1 winding number (the reference's float hierarchy), 2 squared distance, 3 FD gradient (out has 3 doubles per
// point), 4 exact winding number (double sum over all faces), 5 sdf with the exact winding number
void orc_mesh_eval(const double *poly_params, const double *V, int nv, const int *F, int nf, int what, int64_t n,
                   const double *rel, double *out) {
    Shape S = make_mesh_shape(poly_params, V, nv, F, nf);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        const double x = rel[3 * i], y = rel[3 * i + 1], z = rel[3 * i + 2];
        if (what == 0) out[i] = shape_sdf(S, x, y, z);
        else if (what == 1) out[i] = mesh_winding(S, x, y, z);
        else if (what == 2) out[i] = mesh_sqr_distance(S, x, y, z);
        else if (what == 4) out[i] = mesh_winding_exact(S, x, y, z);
        else if (what == 5) out[i] = sd_mesh_exact(S, x, y, z);
        else shape_grad1(S, x, y, z, out + 3 * i);
    }
}
void *orc_create_mesh(const double *poly_params, const double *V, int nv, const int *F, int nf, double weight_p,
                      double safety_hor, double rho, int threads) {
    TrajOptimizerOracle *o = new TrajOptimizerOracle();
    o->sv.shape = make_mesh_shape(poly_params, V, nv, F, nf);
    o->cp.weight_p = weight_p;
    o->cp.safety_hor = safety_hor;
    o->cp.threads = threads > 0 ? threads : 1;
    o->rho = rho;
    return o;
}

// ---- A* front-end collision kernels (frontend_oracle.hpp) ----
void orc_shape_kernels(const char *name, const double *poly_params, int ks, int K, double res, double safeh, double *yaw_out,
                       uint8_t *cells_out, uint8_t *bytes_out) {
    Shape S = make_shape(name, poly_params, nullptr, 0);
    ShapeKernels SK = init_shape_kernels(S, ks, K, res, safeh);
    std::memcpy(yaw_out, SK.yaw.data(), SK.yaw.size() * sizeof(double));
    std::memcpy(cells_out, SK.cells.data(), SK.cells.size());
    std::memcpy(bytes_out, SK.bytes.data(), SK.bytes.size());
}
// free-space map of the whole configuration space: out[k][x][y] = kernelConv(k, (x, y)); variant 0 bool kernels, 1 byte kernels
void orc_cspace(const char *name, const double *poly_params, int ks, int K, double res, double safeh, const uint8_t *occ, int X,
                int Y, int variant, uint8_t *out) {
    Shape S = make_shape(name, poly_params, nullptr, 0);
    ShapeKernels SK = init_shape_kernels(S, ks, K, res, safeh);
    FrontMap M;
    M.build(occ, X, Y, ks);
#pragma omp parallel for collapse(2) schedule(static)
    for (int k = 0; k < K; ++k)
        for (int x = 0; x < X; ++x)
            for (int y = 0; y < Y; ++y)
                out[((size_t)k * X + x) * Y + y] = variant ? kernel_conv_byte(SK, M, k, x, y) : kernel_conv_bool(SK, M, k, x, y);
}
void orc_check_kernel_value(const char *name, const double *poly_params, int ks, int K, double res, double safeh, const uint8_t *occ,
                            int X, int Y, int64_t n, const double *father_yaw, const int *ind_xy, uint8_t *ok_out, double *child_yaw_out) {
    Shape S = make_shape(name, poly_params, nullptr, 0);
    ShapeKernels SK = init_shape_kernels(S, ks, K, res, safeh);
    FrontMap M;
    M.build(occ, X, Y, ks);
    for (int64_t i = 0; i < n; ++i) {
        double cy = father_yaw[i];
        ok_out[i] = check_kernel_value(SK, M, father_yaw[i], cy, ind_xy[2 * i], ind_xy[2 * i + 1]);
        child_yaw_out[i] = cy;
    }
}

// A* neighbour loop for n nodes (front_end_Astar.hpp:192-240): ok / child_yaw / parts are [n][9]
void orc_expand_nodes(const char *name, const double *poly_params, int ks, int K, double res_kernel, double safeh, const uint8_t *occ, int X,
                      int Y, double ox, double oy, double map_res, int64_t n, const int *node_ij, const double *node_yaw, uint8_t *ok_out,
                      double *child_yaw_out, uint8_t *parts_out) {
    Shape S = make_shape(name, poly_params, nullptr, 0);
    ShapeKernels SK = init_shape_kernels(S, ks, K, res_kernel, safeh);
    FrontMap M;
    M.build(occ, X, Y, ks);
    MapGeom G;
    G.ox = ox; G.oy = oy; G.res = map_res;
#pragma omp parallel for schedule(dynamic)
    for (int64_t q = 0; q < n; ++q)
        expand_node(S, SK, M, G, node_ij[2 * q], node_ij[2 * q + 1], node_yaw[q], ks, ok_out + 9 * q, child_yaw_out + 9 * q, parts_out + 9 * q);
}

// PCSmapManager::getPointsInAABB2D (points_in_aabb2d) around (cx, cy): writes up to cap points (x, y), returns how many there are
int64_t orc_points_in_aabb(const uint8_t *occ, int X, int Y, double ox, double oy, double map_res, double cx, double cy, double hbx, double hby,
                           double *xy, int64_t cap) {
    FrontMap M;
    M.build(occ, X, Y, 1);
    MapGeom G;
    G.ox = ox; G.oy = oy; G.res = map_res;
    std::vector<double> pts;
    points_in_aabb2d(M, G, cx, cy, hbx, hby, pts);
    const int64_t np = (int64_t)pts.size() / 2;
    std::memcpy(xy, pts.data(), (size_t)std::min(np, cap) * 2 * sizeof(double));
    return np;
}

// AstarPathSearch for n start/goal pairs; path_out [n][max_path][3], len_out [n] (0 = no path), exp_out [n] expansions
void orc_astar(const char *name, const double *poly_params, int ks, int K, double safeh, const uint8_t *occ, int X, int Y, double ox, double oy,
               double map_res, int n, const double *start_xy, const double *goal_xy, int max_path, double *path_out, int *len_out, int *exp_out) {
    Shape S = make_shape(name, poly_params, nullptr, 0);
    ShapeKernels SK = init_shape_kernels(S, ks, K, map_res, safeh);
    FrontMap M;
    M.build(occ, X, Y, ks);
    MapGeom G;
    G.ox = ox; G.oy = oy; G.res = map_res;
#pragma omp parallel for schedule(dynamic)
    for (int q = 0; q < n; ++q) {
        AstarResult R = astar_search(S, SK, M, G, start_xy + 2 * q, goal_xy + 2 * q);
        const int len = (int)(R.path.size() / 3);
        len_out[q] = (R.success && len <= max_path) ? len : 0;
        exp_out[q] = R.expansions;
        if (len_out[q]) std::memcpy(path_out + (size_t)q * max_path * 3, R.path.data(), R.path.size() * sizeof(double));
    }
}

void *orc_create(const char *name, const double *poly_params, const double *poly_xy, int poly_n, double weight_p,
                 double safety_hor, double rho, int threads) {
    TrajOptimizerOracle *o = new TrajOptimizerOracle();
    o->sv.shape = make_shape(name, poly_params, poly_xy, poly_n);
    o->cp.weight_p = weight_p;
    o->cp.safety_hor = safety_hor;
    o->cp.threads = threads > 0 ? threads : 1;
    o->rho = rho;
    return o;
}
void orc_destroy(void *h) { delete (TrajOptimizerOracle *)h; }
void orc_set_threads(void *h, int threads) { ((TrajOptimizerOracle *)h)->cp.threads = threads > 0 ? threads : 1; }
int orc_max_threads() { return omp_get_max_threads(); }
int orc_num_procs() { return omp_get_num_procs(); }

void orc_set_points(void *h, const double *pts, int64_t P, int stride) {
    TrajOptimizerOracle *o = (TrajOptimizerOracle *)h;
    o->points.resize((size_t)P * 3);
    for (int64_t i = 0; i < P; ++i) {
        o->points[3 * i] = pts[i * stride];
        o->points[3 * i + 1] = pts[i * stride + 1];
        o->points[3 * i + 2] = stride > 2 ? pts[i * stride + 2] : 0.0;
    }
    o->P = P;
}
// updateTraj from MINCO coefficients (6N x 3 col-major) and durations
void orc_set_traj(void *h, int N, const double *T, const double *coeffs) {
    TrajOptimizerOracle *o = (TrajOptimizerOracle *)h;
    Trajectory tr;
    trajectory_from_coeffs(N, T, coeffs, tr);
    o->sv.updateTraj(tr);
}
double orc_traj_duration(void *h) { return ((TrajOptimizerOracle *)h)->sv.traj_duration; }
void orc_traj_pos(void *h, double t, double *p3) { ((TrajOptimizerOracle *)h)->sv.traj.getPos(t, p3); }
void orc_traj_vel(void *h, double t, double *v3) { ((TrajOptimizerOracle *)h)->sv.traj.getVel(t, v3); }
double orc_sdf_at(void *h, const double *p3, double t) { return ((TrajOptimizerOracle *)h)->sv.sdfAt(p3, t); }
double orc_choice_t_init(void *h, const double *p3, double dt) {
    return ((TrajOptimizerOracle *)h)->sv.choiceTInit(p3, dt);
}
void orc_gradient_descent(void *h, const double *p3, double tmin, double tmax, double x0, double *fx, double *x) {
    ((TrajOptimizerOracle *)h)->sv.gradientDescent(tmin, tmax, x0, *fx, *x, p3);
}
// Descent statistics per point (analysis tool for the kernel design, not a parity function): runs choiceTInit + the
// reference's gradientDescent control flow and records the number of outer steps, the total number of halvings
// (candidate evaluations) and a histogram of the accepted halving index (bin 29 = a step in which all 29 failed).
void orc_descent_stats(void *h, int64_t P, const double *pts, int *steps, int *halvings, int64_t *jacc_hist30) {
    TrajOptimizerOracle *o = (TrajOptimizerOracle *)h;
    const SweptVolume &sv = o->sv;
    for (int b = 0; b < 30; ++b) jacc_hist30[b] = 0;
    for (int64_t i = 0; i < P; ++i) {
        double p[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
        double ts = sv.choiceTInit(p, 0.15);
        double t_min = std::max(0.0, ts - 3.4), t_max = std::min(ts + 3.4, sv.traj_duration);
        double x = ts, prev_x = 10000000.0, fx = 0, tau;
        int iter = 0, ns = 0, nh = 0;
        bool stop = false;
        while (iter < 1000 && !stop && std::abs(x - prev_x) > 1e-16) {
            if (iter == 0) fx = sv.sdfAt(p, x);
            double g = sv.sdfDotAt(p, x);
            tau = 0.01;
            prev_x = x;
            ns++;
            int acc = 29;
            for (int div = 1; div < 30; div++) {
                iter++;
                nh++;
                double xc = std::max(std::min(x + (-tau * ((int)(g > 0) - (g < 0))), t_max), t_min);
                double fc = sv.sdfAt(p, xc);
                if ((fc - fx) < 0) { x = xc; fx = fc; acc = div - 1; break; }
                tau = 0.5 * tau;
                if (div == 29) stop = true;
            }
            jacc_hist30[acc]++;
        }
        steps[i] = ns;
        halvings[i] = nh;
    }
}
void orc_count_evals(void *h, int on) {
    TrajOptimizerOracle *o = (TrajOptimizerOracle *)h;
    o->sv.count_evals = on != 0;
    o->sv.eval_count = 0;
}
uint64_t orc_eval_count(void *h) { return ((TrajOptimizerOracle *)h)->sv.eval_count; }

// getSDFofSweptVolume<false,true> (A6) per point; pts stride 3 (z used as given)
void orc_query_outer(void *h, int64_t P, const double *pts, double *sdf, double *tstar, double *grad3) {
    TrajOptimizerOracle *o = (TrajOptimizerOracle *)h;
#pragma omp parallel for num_threads(o->cp.threads) schedule(dynamic)
    for (int64_t i = 0; i < P; ++i) {
        double p[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
        double g[3], ts = 0;
        sdf[i] = o->sv.getSDFofSweptVolume(p, ts, g);
        tstar[i] = ts;
        grad3[3 * i] = g[0]; grad3[3 * i + 1] = g[1]; grad3[3 * i + 2] = g[2];
    }
}
// getTrueSDFofSweptVolume<true> (A7) per point (raw outputs: world-frame direction when sdf <= 0)
void orc_query(void *h, int64_t P, const double *pts, double *sdf, double *tstar, double *grad3, int *rounds) {
    TrajOptimizerOracle *o = (TrajOptimizerOracle *)h;
#pragma omp parallel for num_threads(o->cp.threads) schedule(dynamic)
    for (int64_t i = 0; i < P; ++i) {
        double p[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
        double g[3], ts = 0;
        int r = 0;
        sdf[i] = o->sv.getTrueSDFofSweptVolume(p, ts, g, &r);
        tstar[i] = ts;
        grad3[3 * i] = g[0]; grad3[3 * i + 1] = g[1]; grad3[3 * i + 2] = g[2];
        if (rounds) rounds[i] = r;
    }
}

// addSaftyPenaOnSweptVolumeParallelTrueSDF (accumulating). per_point: P x 7 doubles
// (sdf, tstar, gx, gy, gz, piece, pena) or NULL. Returns number of points that took the GSIP branch.
int64_t orc_cost_grad(void *h, int N, const double *T, const double *coeffs, double *cost_io, double *gradT_io,
                      double *gradC_io, double *per_point) {
    TrajOptimizerOracle *o = (TrajOptimizerOracle *)h;
    Trajectory tr;
    trajectory_from_coeffs(N, T, coeffs, tr);
    o->sv.updateTraj(tr);
    std::vector<PointResult> pr;
    if (per_point) pr.resize(o->P);
    int64_t inside = 0;
    addSafetyPenaltyTrueSDF(o->sv, o->cp, N, T, coeffs, o->points.data(), o->P, 3, *cost_io, gradT_io, gradC_io,
                            per_point ? pr.data() : nullptr, &inside);
    if (per_point)
        for (int64_t i = 0; i < o->P; ++i) {
            double *r = per_point + 7 * i;
            r[0] = pr[i].sdf; r[1] = pr[i].tstar; r[2] = pr[i].g[0]; r[3] = pr[i].g[1]; r[4] = pr[i].g[2];
            r[5] = pr[i].piece; r[6] = pr[i].pena;
        }
    return inside;
}

// timed variant used by bench.py (returns seconds, best of `reps` after `warm` warm-ups)
double orc_time_cost_grad(void *h, int N, const double *T, const double *coeffs, int warm, int reps,
                          double *cost_out) {
    TrajOptimizerOracle *o = (TrajOptimizerOracle *)h;
    std::vector<double> gT(N), gC((size_t)18 * N);
    double best = 1e300;
    for (int r = 0; r < warm + reps; ++r) {
        double cost = 0;
        std::fill(gT.begin(), gT.end(), 0.0);
        std::fill(gC.begin(), gC.end(), 0.0);
        double t0 = omp_get_wtime();
        orc_cost_grad(h, N, T, coeffs, &cost, gT.data(), gC.data(), nullptr);
        double dt = omp_get_wtime() - t0;
        if (r >= warm && dt < best) best = dt;
        if (cost_out) *cost_out = cost;
    }
    (void)o;
    return best;
}

// MINCO_S3NU: setConditions + setParameters; outputs b (6N x 3), energy, dE/dc, dE/dT
void orc_minco_forward(const double *initS, const double *finalS, int N, const double *q, const double *T,
                       double *b_out, double *energy, double *gdC, double *gdT) {
    MincoS3NU m;
    m.setConditions(initS, finalS, N);
    m.setParameters(q, T);
    std::memcpy(b_out, m.b.data(), sizeof(double) * 18 * N);
    if (energy) *energy = m.getEnergy();
    if (gdC) m.getEnergyPartialGradByCoeffs(gdC);
    if (gdT) m.getEnergyPartialGradByTimes(gdT);
}
// MINCO_S3NU::propogateGrad
void orc_minco_propagate(const double *initS, const double *finalS, int N, const double *q, const double *T,
                         const double *gdC, const double *gdT, double *gradQ, double *gradT) {
    MincoS3NU m;
    m.setConditions(initS, finalS, N);
    m.setParameters(q, T);
    m.propogateGrad(gdC, gdT, gradQ, gradT);
}
// smoothedL1 (back_end_optimizer.hpp:316-340) over n samples; ret[i] = its boolean return
void orc_smoothed_l1(int64_t n, const double *x, double mu, double *f, double *df, uint8_t *ret) {
    for (int64_t i = 0; i < n; ++i) {
        double ff = 0, dd = 0;
        ret[i] = smoothedL1(x[i], mu, ff, dd) ? 1 : 0;
        f[i] = ff; df[i] = dd;
    }
}
void orc_forward_T(int n, const double *tau, double *T) { for (int i = 0; i < n; ++i) T[i] = forwardT1(tau[i]); }
void orc_backward_T(int n, const double *T, double *tau) { for (int i = 0; i < n; ++i) tau[i] = backwardT1(T[i]); }

void orc_set_conditions(void *h, const double *initS, const double *finalS, int N) {
    ((TrajOptimizerOracle *)h)->setConditions(initS, finalS, N);
}
// costFunctionLmbmParallel(ptr, x, g, n)
double orc_evaluate(void *h, const double *x, double *g, int n) {
    (void)n;
    return ((TrajOptimizerOracle *)h)->evaluate(x, g);
}
void orc_last_costs(void *h, double *out3) {
    TrajOptimizerOracle *o = (TrajOptimizerOracle *)h;
    out3[0] = o->cost_pos; out3[1] = o->cost_other; out3[2] = o->cost_total;
}
void orc_get_coeffs(void *h, double *T_out, double *b_out) {
    TrajOptimizerOracle *o = (TrajOptimizerOracle *)h;
    std::memcpy(T_out, o->times.data(), sizeof(double) * o->pieceN);
    std::memcpy(b_out, o->minco.b.data(), sizeof(double) * 18 * o->pieceN);
}

// L-BFGS (lbfgs_ref.hpp) driving orc_evaluate. stats_out: [final f, iterations, evaluations, seconds]
int orc_lbfgs(void *h, double *x, int n, int mem_size, int past, double delta, double g_epsilon, int max_iterations,
              double min_step, double *stats_out) {
    TrajOptimizerOracle *o = (TrajOptimizerOracle *)h;
    LbfgsParams p;
    p.mem_size = mem_size; p.past = past; p.delta = delta; p.g_epsilon = g_epsilon;
    p.max_iterations = max_iterations; p.min_step = min_step;
    std::vector<double> xv(x, x + n);
    double f = 0;
    int iters = 0;
    o->n_evals = 0;
    double t0 = omp_get_wtime();
    int ret = lbfgs_optimize(xv, f, [&](const double *xx, double *gg) { return o->evaluate(xx, gg); }, nullptr, p,
                             &iters);
    double dt = omp_get_wtime() - t0;
    std::memcpy(x, xv.data(), sizeof(double) * n);
    if (stats_out) { stats_out[0] = f; stats_out[1] = iters; stats_out[2] = (double)o->n_evals; stats_out[3] = dt; }
    return ret;
}

// Generic L-BFGS over a C callback (used to test the host L-BFGS of the product on analytic functions)
typedef double (*orc_eval_cb)(void *inst, const double *x, double *g, int n);
int orc_lbfgs_cb(orc_eval_cb cb, void *inst, double *x, int n, int mem_size, int past, double delta,
                 double g_epsilon, int max_iterations, double *stats_out) {
    LbfgsParams p;
    p.mem_size = mem_size; p.past = past; p.delta = delta; p.g_epsilon = g_epsilon; p.max_iterations = max_iterations;
    std::vector<double> xv(x, x + n);
    double f = 0;
    int iters = 0, evals = 0;
    int ret = lbfgs_optimize(xv, f, [&](const double *xx, double *gg) { ++evals; return cb(inst, xx, gg, n); },
                             nullptr, p, &iters);
    std::memcpy(x, xv.data(), sizeof(double) * n);
    if (stats_out) { stats_out[0] = f; stats_out[1] = iters; stats_out[2] = evals; }
    return ret;
}

}  // extern "C"
