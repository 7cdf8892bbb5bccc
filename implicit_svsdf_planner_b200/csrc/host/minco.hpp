// host/minco.hpp — minimum-jerk (s = 3) non-uniform MINCO spline, its energy and the adjoint that maps d/d(coefficients, durations)
// back to d/d(waypoints, durations).
//
// Same mathematics and public surface as the reference's MINCO_S3NU
// (src/utils/include/utils/minco.hpp:397-655: setConditions / setParameters / getEnergy /
// getEnergyPartialGradByCoeffs / getEnergyPartialGradByTimes / propogateGrad), written without Eigen.
// The 6N x 6N system is banded (half-bandwidth 6); it is stored row-wise in a dense band and eliminated without
// pivoting, which the structure of the system permits (the reference does the same, minco.hpp:99-131).
// The arithmetic is SVSDF_HD functions over caller-provided arrays (MincoView), so the device back end (svsdf_backend.cu) runs the
// same code as the host classes below, which own their storage.
#pragma once
#include <cmath>
#include <cstring>
#include <vector>

#include "../svsdf_types.h"

namespace svsdf {
namespace host {

constexpr int kBandBW = 6;
constexpr int kBandW = 2 * kBandBW + 1;

// The lanes that share one problem's independent work: rows of one elimination step, the three right-hand sides, pieces.  Each
// element sees the same operations in the same order whatever the team, so every team gives the same bits.  The host runs one lane
// (SerialTeam); the device back end a warp (svsdf_backend.cu).  sync(): every lane's writes are visible to the others.
struct SerialTeam {
    SVSDF_HD int lane() const { return 0; }
    SVSDF_HD int size() const { return 1; }
    SVSDF_HD void sync() const {}
};

SVSDF_HD inline int band_imin(int a, int b) { return b < a ? b : a; }
SVSDF_HD inline int band_imax(int a, int b) { return a < b ? b : a; }
// element (r, c) of a band matrix stored row-wise, kBandW doubles per row
SVSDF_HD inline double &band_at(double *a, int r, int c) { return a[(size_t)r * kBandW + (c - r + kBandBW)]; }
SVSDF_HD inline double band_at(const double *a, int r, int c) { return a[(size_t)r * kBandW + (c - r + kBandBW)]; }

// In-place LU (Doolittle, unit lower), no pivoting.  The rows below one pivot are independent: one lane each.
template <class Team = SerialTeam>
SVSDF_HD inline void band_factorize(double *a, int n, const Team &team = Team()) {
    for (int k = 0; k < n - 1; ++k) {
        const double piv = band_at(a, k, k);
        const int rmax = band_imin(k + kBandBW, n - 1);
        const int cmax = band_imin(k + kBandBW, n - 1);
        for (int r = k + 1 + team.lane(); r <= rmax; r += team.size()) {
            double &l = band_at(a, r, k);
            if (l == 0.0) continue;
            l /= piv;
            for (int c = k + 1; c <= cmax; ++c) {
                const double u = band_at(a, k, c);
                if (u != 0.0) band_at(a, r, c) -= l * u;
            }
        }
        team.sync();
    }
}
// Solve A x = b for the right-hand side b (n), overwritten by x.
SVSDF_HD inline void band_solve1(const double *a, int n, double *b) {
    for (int j = 0; j < n; ++j) {
        const int rmax = band_imin(j + kBandBW, n - 1);
        const double bj = b[j];
        for (int r = j + 1; r <= rmax; ++r) {
            const double l = band_at(a, r, j);
            if (l != 0.0) b[r] -= l * bj;
        }
    }
    for (int j = n - 1; j >= 0; --j) {
        b[j] /= band_at(a, j, j);
        const int rmin = band_imax(0, j - kBandBW);
        const double bj = b[j];
        for (int r = rmin; r < j; ++r) {
            const double u = band_at(a, r, j);
            if (u != 0.0) b[r] -= u * bj;
        }
    }
}
// Solve A^T x = b.
SVSDF_HD inline void band_solve1_transposed(const double *a, int n, double *b) {
    for (int j = 0; j < n; ++j) {  // U^T is lower triangular
        b[j] /= band_at(a, j, j);
        const int cmax = band_imin(j + kBandBW, n - 1);
        const double bj = b[j];
        for (int i = j + 1; i <= cmax; ++i) {
            const double u = band_at(a, j, i);
            if (u != 0.0) b[i] -= u * bj;
        }
    }
    for (int j = n - 1; j >= 0; --j) {  // L^T is unit upper triangular
        const int cmin = band_imax(0, j - kBandBW);
        const double bj = b[j];
        for (int i = cmin; i < j; ++i) {
            const double l = band_at(a, j, i);
            if (l != 0.0) b[i] -= l * bj;
        }
    }
}

// Solve A X = B (transposed: A^T X = B) for the three right-hand sides of B (n x 3 column-major), one lane each.
template <class Team = SerialTeam>
SVSDF_HD inline void band_solve3(const double *a, int n, double *B, bool transposed, const Team &team = Team()) {
    for (int c = team.lane(); c < 3; c += team.size()) {
        if (transposed) band_solve1_transposed(a, n, B + (size_t)c * n);
        else band_solve1(a, n, B + (size_t)c * n);
    }
    team.sync();
}

class BandMatrix {
   public:
    static constexpr int BW = kBandBW;
    static constexpr int W = kBandW;
    void resize(int n) {
        n_ = n;
        a_.assign((size_t)n * W, 0.0);
    }
    void zero() { std::fill(a_.begin(), a_.end(), 0.0); }
    inline double &at(int r, int c) { return band_at(a_.data(), r, c); }
    inline double at(int r, int c) const { return band_at(a_.data(), r, c); }
    int n() const { return n_; }
    double *data() { return a_.data(); }
    const double *data() const { return a_.data(); }

    void factorize() { band_factorize(a_.data(), n_); }
    // Solve A X = B for m right-hand sides; B is n x m column-major (B[c*n + r]), overwritten by X.
    void solve(double *B, int m) const {
        for (int c = 0; c < m; ++c) band_solve1(a_.data(), n_, B + (size_t)c * n_);
    }
    // Solve A^T X = B.
    void solve_transposed(double *B, int m) const {
        for (int c = 0; c < m; ++c) band_solve1_transposed(a_.data(), n_, B + (size_t)c * n_);
    }

   private:
    int n_ = 0;
    std::vector<double> a_;
};

// One MINCO_S3NU of N pieces on caller-provided storage: head / tail 3x3 column-major (column k = k-th derivative), A the band
// (6N x kBandW), b the coefficients (6N x 3 column-major, offset d*6N + 6i + k), t the powers T^1..T^5 of every duration (5N).
struct MincoView {
    int N;
    const double *head, *tail;
    double *A, *b, *t;
};
SVSDF_HD inline size_t minco_band_doubles(int N) { return (size_t)6 * N * kBandW; }

SVSDF_HD inline void minco_fill_system(const MincoView &V, const double *inPs);
// setParameters: inPs 3 x (N-1) column-major, ts N durations.  Zeroes and fills the system, factorises it and solves for b.
template <class Team = SerialTeam>
SVSDF_HD inline void minco_set_parameters(const MincoView &V, const double *inPs, const double *ts, const Team &team = Team()) {
    const int N = V.N, n = 6 * N;
    double *A = V.A, *b = V.b;
    for (int i = team.lane(); i < N; i += team.size()) {
        double *p = V.t + 5 * i;
        p[0] = ts[i];
        p[1] = p[0] * p[0];
        p[2] = p[1] * p[0];
        p[3] = p[1] * p[1];
        p[4] = p[3] * p[0];
    }
    for (size_t e = team.lane(); e < minco_band_doubles(N); e += team.size()) A[e] = 0.0;
    for (int e = team.lane(); e < 3 * n; e += team.size()) b[e] = 0.0;
    team.sync();
    if (team.lane() == 0) minco_fill_system(V, inPs);
    team.sync();
    band_factorize(A, n, team);
    band_solve3(A, n, b, false, team);
}
// the system of setParameters (after the powers of the durations, into a zeroed band and right-hand side)
SVSDF_HD inline void minco_fill_system(const MincoView &V, const double *inPs) {
    const int N = V.N, n = 6 * N;
    double *A = V.A, *b = V.b;
    // head: position, velocity, acceleration
    band_at(A, 0, 0) = 1.0;
    band_at(A, 1, 1) = 1.0;
    band_at(A, 2, 2) = 2.0;
    for (int d = 0; d < 3; ++d)
        for (int k = 0; k < 3; ++k) b[d * n + k] = V.head[k * 3 + d];
    for (int i = 0; i < N - 1; ++i) {
        const double *p = V.t + 5 * i;
        const double T1 = p[0], T2 = p[1], T3 = p[2], T4 = p[3], T5 = p[4];
        const int r = 6 * i;
        // jerk, snap continuity
        band_at(A, r + 3, r + 3) = 6.0;  band_at(A, r + 3, r + 4) = 24.0 * T1;  band_at(A, r + 3, r + 5) = 60.0 * T2;  band_at(A, r + 3, r + 9) = -6.0;
        band_at(A, r + 4, r + 4) = 24.0; band_at(A, r + 4, r + 5) = 120.0 * T1; band_at(A, r + 4, r + 10) = -24.0;
        // waypoint, position continuity
        const double pw[6] = {1.0, T1, T2, T3, T4, T5};
        for (int k = 0; k < 6; ++k) { band_at(A, r + 5, r + k) = pw[k]; band_at(A, r + 6, r + k) = pw[k]; }
        band_at(A, r + 6, r + 6) = -1.0;
        // velocity, acceleration continuity
        band_at(A, r + 7, r + 1) = 1.0; band_at(A, r + 7, r + 2) = 2 * T1; band_at(A, r + 7, r + 3) = 3 * T2; band_at(A, r + 7, r + 4) = 4 * T3; band_at(A, r + 7, r + 5) = 5 * T4; band_at(A, r + 7, r + 7) = -1.0;
        band_at(A, r + 8, r + 2) = 2.0; band_at(A, r + 8, r + 3) = 6 * T1; band_at(A, r + 8, r + 4) = 12 * T2; band_at(A, r + 8, r + 5) = 20 * T3; band_at(A, r + 8, r + 8) = -2.0;
        for (int d = 0; d < 3; ++d) b[d * n + r + 5] = inPs[i * 3 + d];
    }
    {
        const double *p = V.t + 5 * (N - 1);
        const double T1 = p[0], T2 = p[1], T3 = p[2], T4 = p[3], T5 = p[4];
        const int r = n - 6;
        const double pw[6] = {1.0, T1, T2, T3, T4, T5};
        for (int k = 0; k < 6; ++k) band_at(A, n - 3, r + k) = pw[k];
        band_at(A, n - 2, r + 1) = 1.0; band_at(A, n - 2, r + 2) = 2 * T1; band_at(A, n - 2, r + 3) = 3 * T2; band_at(A, n - 2, r + 4) = 4 * T3; band_at(A, n - 2, r + 5) = 5 * T4;
        band_at(A, n - 1, r + 2) = 2.0; band_at(A, n - 1, r + 3) = 6 * T1; band_at(A, n - 1, r + 4) = 12 * T2; band_at(A, n - 1, r + 5) = 20 * T3;
        for (int d = 0; d < 3; ++d)
            for (int k = 0; k < 3; ++k) b[d * n + n - 3 + k] = V.tail[k * 3 + d];
    }
}
SVSDF_HD inline double minco_dot(const MincoView &V, int i, int r1, int r2) {
    const int n = 6 * V.N;
    double s = 0.0;
    for (int d = 0; d < 3; ++d) s += V.b[(size_t)d * n + 6 * i + r1] * V.b[(size_t)d * n + 6 * i + r2];
    return s;
}
SVSDF_HD inline double minco_energy(const MincoView &V) {
    double e = 0.0;
    for (int i = 0; i < V.N; ++i) {
        const double *p = V.t + 5 * i;
        e += 36.0 * minco_dot(V, i, 3, 3) * p[0] + 144.0 * minco_dot(V, i, 4, 3) * p[1] + 192.0 * minco_dot(V, i, 4, 4) * p[2] +
             240.0 * minco_dot(V, i, 5, 3) * p[2] + 720.0 * minco_dot(V, i, 5, 4) * p[3] + 720.0 * minco_dot(V, i, 5, 5) * p[4];
    }
    return e;
}
template <class Team = SerialTeam>
SVSDF_HD inline void minco_energy_grad_coeffs(const MincoView &V, double *gdC, const Team &team = Team()) {
    const int n = 6 * V.N;
    for (int i = team.lane(); i < V.N; i += team.size()) {
        const double *p = V.t + 5 * i;
        for (int d = 0; d < 3; ++d) {
            const double *c = V.b + (size_t)d * n + 6 * i;
            double *g = gdC + (size_t)d * n + 6 * i;
            g[0] = g[1] = g[2] = 0.0;
            g[3] = 72.0 * c[3] * p[0] + 144.0 * c[4] * p[1] + 240.0 * c[5] * p[2];
            g[4] = 144.0 * c[3] * p[1] + 384.0 * c[4] * p[2] + 720.0 * c[5] * p[3];
            g[5] = 240.0 * c[3] * p[2] + 720.0 * c[4] * p[3] + 1440.0 * c[5] * p[4];
        }
    }
}
template <class Team = SerialTeam>
SVSDF_HD inline void minco_energy_grad_times(const MincoView &V, double *gdT, const Team &team = Team()) {
    for (int i = team.lane(); i < V.N; i += team.size()) {
        const double *p = V.t + 5 * i;
        gdT[i] = 36.0 * minco_dot(V, i, 3, 3) + 288.0 * minco_dot(V, i, 4, 3) * p[0] + 576.0 * minco_dot(V, i, 4, 4) * p[1] +
                 720.0 * minco_dot(V, i, 5, 3) * p[1] + 2880.0 * minco_dot(V, i, 5, 4) * p[2] + 3600.0 * minco_dot(V, i, 5, 5) * p[3];
    }
}
// propogateGrad: adj (18N) is scratch; gradByPoints 3 x (N-1) column-major, gradByTimes N.
template <class Team = SerialTeam>
SVSDF_HD inline void minco_propagate(const MincoView &V, const double *partialGradByCoeffs, const double *partialGradByTimes, double *adj,
                                     double *gradByPoints, double *gradByTimes, const Team &team = Team()) {
    const int N = V.N, n = 6 * N;
    for (int e = team.lane(); e < 3 * n; e += team.size()) adj[e] = partialGradByCoeffs[e];
    team.sync();
    band_solve3(V.A, n, adj, true, team);
    for (int i = team.lane(); i < N - 1; i += team.size())
        for (int d = 0; d < 3; ++d) gradByPoints[i * 3 + d] = adj[(size_t)d * n + 6 * i + 5];
    for (int i = team.lane(); i < N; i += team.size()) {
        const double *p = V.t + 5 * i;
        const double T1 = p[0], T2 = p[1], T3 = p[2], T4 = p[3];
        double s = 0.0;
        for (int d = 0; d < 3; ++d) {
            const double *c = V.b + (size_t)d * n + 6 * i;
            const double nvel = -(c[1] + 2.0 * T1 * c[2] + 3.0 * T2 * c[3] + 4.0 * T3 * c[4] + 5.0 * T4 * c[5]);
            const double nacc = -(2.0 * c[2] + 6.0 * T1 * c[3] + 12.0 * T2 * c[4] + 20.0 * T3 * c[5]);
            const double njer = -(6.0 * c[3] + 24.0 * T1 * c[4] + 60.0 * T2 * c[5]);
            if (i < N - 1) {
                const double nsna = -(24.0 * c[4] + 120.0 * T1 * c[5]);
                const double ncra = -120.0 * c[5];
                const double *a = adj + (size_t)d * n + 6 * i + 3;
                // rows 6i+3..6i+8: jerk, snap, waypoint, position, velocity, acceleration constraints
                s += nsna * a[0] + ncra * a[1] + nvel * a[2] + nvel * a[3] + nacc * a[4] + njer * a[5];
            } else {
                const double *a = adj + (size_t)d * n + n - 3;
                s += nvel * a[0] + nacc * a[1] + njer * a[2];
            }
        }
        gradByTimes[i] = s + partialGradByTimes[i];
    }
    team.sync();
}

class MincoS3NU {
   public:
    void setConditions(const double *headState, const double *tailState, int pieceNum) {
        N_ = pieceNum;
        std::memcpy(head_, headState, sizeof(head_));
        std::memcpy(tail_, tailState, sizeof(tail_));
        A_.resize(6 * N_);
        b_.assign((size_t)18 * N_, 0.0);
        t_.assign((size_t)5 * N_, 0.0);
    }
    int pieces() const { return N_; }
    // inPs: 3 x (N-1) column-major; ts: N durations.
    void setParameters(const double *inPs, const double *ts) { minco_set_parameters(view(), inPs, ts); }
    // MINCO coefficient matrix b: 6N x 3, column-major (offset d*6N + 6i + k)
    const double *getCoeffs() const { return b_.data(); }
    const double *durations5() const { return t_.data(); }

    double getEnergy() const { return minco_energy(view()); }
    void getEnergyPartialGradByCoeffs(double *gdC) const { minco_energy_grad_coeffs(view(), gdC); }
    void getEnergyPartialGradByTimes(double *gdT) const { minco_energy_grad_times(view(), gdT); }
    // propogateGrad: gradByPoints 3 x (N-1) column-major, gradByTimes N.
    void propogateGrad(const double *partialGradByCoeffs, const double *partialGradByTimes, double *gradByPoints,
                       double *gradByTimes) const {
        adj_.assign((size_t)18 * N_, 0.0);
        minco_propagate(view(), partialGradByCoeffs, partialGradByTimes, adj_.data(), gradByPoints, gradByTimes);
    }

    // the object's arrays (setConditions sized them); the const methods only read through it
    MincoView view() const {
        return MincoView{N_, head_, tail_, const_cast<double *>(A_.data()), const_cast<double *>(b_.data()), const_cast<double *>(t_.data())};
    }

   private:
    int N_ = 0;
    double head_[9], tail_[9];
    BandMatrix A_;
    std::vector<double> b_, t_;
    mutable std::vector<double> adj_;
};

// tau <-> T diffeomorphism (back_end_optimizer.hpp:199-289)
SVSDF_HD inline double forwardT(double tau) {
    return tau > 0.0 ? ((0.5 * tau + 1.0) * tau + 1.0) : 1.0 / ((0.5 * tau - 1.0) * tau + 1.0);
}
inline double backwardT(double T) { return T > 1.0 ? (std::sqrt(2.0 * T - 1.0) - 1.0) : (1.0 - std::sqrt(2.0 / T - 1.0)); }
SVSDF_HD inline double backwardGradT(double tau, double gradT) {
    if (tau > 0) return gradT * (tau + 1.0);
    const double den = (0.5 * tau - 1.0) * tau + 1.0;
    return gradT * (1.0 - tau) / (den * den);
}

// Speed and yaw-rate limits (svsdf_set_dynamics): the yaml's vmax, omgmax, weight_v, weight_omg, smoothingEps and integralIntervs.
struct DynamicsParams {
    double vmax, omgmax, weight_v, weight_omg, eps;
    int res;  // integralIntervs: samples j = 0 .. res per piece
};
// smoothedL1 (back_end_optimizer.hpp:316-340): false below 0, the cubic on [0, mu], x - mu / 2 above
SVSDF_HD inline bool smoothed_l1(double x, double mu, double &f, double &df) {
    if (x < 0.0) return false;
    if (x > mu) {
        f = x - 0.5 * mu;
        df = 1.0;
        return true;
    }
    const double xdmu = x / mu;
    const double sqrxdmu = xdmu * xdmu;
    const double mumxd2 = mu - 0.5 * x;
    f = mumxd2 * sqrxdmu * xdmu;
    df = sqrxdmu * ((-0.5) * xdmu + 3.0 * mumxd2 / mu);
    return true;
}
// The dynamics penalty: the reference's addTimeIntPenalty (back_end_optimizer.hpp:411-533) with the two violations it computes,
// violaVel = |vel_xy|^2 - vmax^2 and violaOmg = vel_yaw^2 - omgmax^2, penalised through smoothed_l1 (the reference computes them and
// penalises neither).  No St(t) term: the limits are on the body's path, not on its shape.  b: MINCO coefficients (6N x 3
// column-major), T: durations.  Adds the partials to gradC (6N x 3) and gradT (N), writes each piece's cost to partial (N) and returns
// the cost (every lane).  Per piece i: step = T_i * (1 / res) as the reference computes it; at s = j step, j = 0 .. res ascending,
// vel = beta1(s)^T c_i and acc = beta2(s)^T c_i (each a left-to-right sum over k = 1 .. 5, resp. 2 .. 5), node = 0.5 at j = 0 and
// j = res else 1, alpha = j * (1 / res).  A sample where neither violation is >= 0 adds nothing; otherwise gradVel = (w_v df_v 2 vel_x,
// w_v df_v 2 vel_y, w_omg df_omg 2 vel_yaw) (a zero where its violation is below 0), pena = w_v f_v + w_omg f_omg, and
//   gradC[d][k] += beta1_k gradVel_d node step  (k = 1 .. 5; beta1_0 = 0)
//   gradT[i]    += (gradVel . acc) alpha node step + node (1 / res) pena
//   partial[i]  += node step pena
// Summation order: within a piece the samples in ascending j, into the piece's partial (from 0.0); the cost is then the sum of the
// partials in ascending i.  One lane owns a piece's samples, so every team gives the same bits.
template <class Team = SerialTeam>
SVSDF_HD inline double dynamics_penalty(const DynamicsParams &p, int N, const double *T, const double *b, double *gradC, double *gradT,
                                        double *partial, const Team &team = Team()) {
    const int n = 6 * N, res = p.res;
    const double velSqrMax = p.vmax * p.vmax, omgSqrMax = p.omgmax * p.omgmax, integralFrac = 1.0 / res;
    for (int i = team.lane(); i < N; i += team.size()) {
        const double step = T[i] * integralFrac;
        double part = 0.0;
        for (int j = 0; j <= res; ++j) {
            // beta1 = (0, 1, 2 s1, 3 s2, 4 s3, 5 s4), beta2 = (0, 0, 2, 6 s1, 12 s2, 20 s3), formed where they are used
            const double s1 = j * step, s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2;
            double vel[3];
            for (int d = 0; d < 3; ++d) {
                const double *c = b + (size_t)d * n + 6 * i;
                vel[d] = c[1] + 2.0 * s1 * c[2] + 3.0 * s2 * c[3] + 4.0 * s3 * c[4] + 5.0 * s4 * c[5];
            }
            const double violaVel = vel[0] * vel[0] + vel[1] * vel[1] - velSqrMax;
            const double violaOmg = vel[2] * vel[2] - omgSqrMax;
            double f, df, pena = 0.0, gradVel[3] = {0.0, 0.0, 0.0};
            bool active = false;
            if (smoothed_l1(violaVel, p.eps, f, df)) {
                gradVel[0] = p.weight_v * df * 2.0 * vel[0];
                gradVel[1] = p.weight_v * df * 2.0 * vel[1];
                pena += p.weight_v * f;
                active = true;
            }
            if (smoothed_l1(violaOmg, p.eps, f, df)) {
                gradVel[2] = p.weight_omg * df * 2.0 * vel[2];
                pena += p.weight_omg * f;
                active = true;
            }
            if (!active) continue;
            const double node = (j == 0 || j == res) ? 0.5 : 1.0, alpha = j * integralFrac;
            double dot = 0.0;
            for (int d = 0; d < 3; ++d) {
                const double *c = b + (size_t)d * n + 6 * i;
                double *g = gradC + (size_t)d * n + 6 * i;
                const double acc = 2.0 * c[2] + 6.0 * s1 * c[3] + 12.0 * s2 * c[4] + 20.0 * s3 * c[5];
                dot = d == 0 ? gradVel[0] * acc : dot + gradVel[d] * acc;
                g[1] += 1.0 * gradVel[d] * node * step;
                g[2] += 2.0 * s1 * gradVel[d] * node * step;
                g[3] += 3.0 * s2 * gradVel[d] * node * step;
                g[4] += 4.0 * s3 * gradVel[d] * node * step;
                g[5] += 5.0 * s4 * gradVel[d] * node * step;
            }
            gradT[i] += dot * alpha * node * step + node * integralFrac * pena;
            part += node * step * pena;
        }
        partial[i] = part;
    }
    team.sync();
    double cost = 0.0;
    for (int i = 0; i < N; ++i) cost += partial[i];
    return cost;
}

// The pose-sampled obstacle penalty (svsdf_set_pose_penalty): weight_p and integralIntervs of addTimeIntPenalty's grad_cost_p term.
struct PoseParams {
    double weight;
    int res;  // integralIntervs: samples j = 0 .. res per piece
};
// The chain rule of the pose penalty: addTimeIntPenalty's (back_end_optimizer.hpp:411-533) use of grad_cost_p (:956-1028), which the
// reference computes and never applies.  rec: the per-sample records (costp, gradp_x, gradp_y, grad_yaw) the pose kernel wrote
// (svsdf_pose.cu), N (res + 1) of them, piece-major.  b, T, gradC, gradT, partial and the return value as dynamics_penalty's; step,
// s, node and alpha too.  A sample is active when costp > 0; then gP = weight (gradp_x, gradp_y, grad_yaw), pena = weight costp, and
//   gradC[d][k] += beta0_k gP_d node step  (beta0 = (1, s, s^2, .., s^5))
//   gradT[i]    += (gP . vel) alpha node step + node (1 / res) pena,  vel = beta1(s)^T c_i
//   partial[i]  += node step pena
// An inactive sample adds nothing.  Summation order as dynamics_penalty's: one lane owns a piece, its samples in ascending j, then the
// partials in ascending i.
template <class Team = SerialTeam>
SVSDF_HD inline double pose_penalty(const PoseParams &p, int N, const double *T, const double *b, const double *rec, double *gradC,
                                    double *gradT, double *partial, const Team &team = Team()) {
    const int n = 6 * N, res = p.res;
    const double integralFrac = 1.0 / res;
    for (int i = team.lane(); i < N; i += team.size()) {
        const double step = T[i] * integralFrac;
        double part = 0.0;
        for (int j = 0; j <= res; ++j) {
            const double *r = rec + 4 * ((size_t)i * (res + 1) + j);
            if (!(r[0] > 0.0)) continue;
            const double gP[3] = {p.weight * r[1], p.weight * r[2], p.weight * r[3]}, pena = p.weight * r[0];
            const double s1 = j * step, s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2, s5 = s4 * s1;
            const double node = (j == 0 || j == res) ? 0.5 : 1.0, alpha = j * integralFrac;
            double dot = 0.0;
            for (int d = 0; d < 3; ++d) {
                const double *c = b + (size_t)d * n + 6 * i;
                double *g = gradC + (size_t)d * n + 6 * i;
                const double vel = c[1] + 2.0 * s1 * c[2] + 3.0 * s2 * c[3] + 4.0 * s3 * c[4] + 5.0 * s4 * c[5];
                dot = d == 0 ? gP[0] * vel : dot + gP[d] * vel;
                g[0] += 1.0 * gP[d] * node * step;
                g[1] += s1 * gP[d] * node * step;
                g[2] += s2 * gP[d] * node * step;
                g[3] += s3 * gP[d] * node * step;
                g[4] += s4 * gP[d] * node * step;
                g[5] += s5 * gP[d] * node * step;
            }
            gradT[i] += dot * alpha * node * step + node * integralFrac * pena;
            part += node * step * pena;
        }
        partial[i] = part;
    }
    team.sync();
    double cost = 0.0;
    for (int i = 0; i < N; ++i) cost += partial[i];
    return cost;
}

// The host half of one back-end evaluation (back_end_optimizer.hpp:353-398) on flat storage of N pieces: times, gradByTimes,
// partialGradByTimes (N each), partialGradByCoeffs and adj (18N each), gradByPoints (3 (N - 1)), dynPartial (N: the pose and the
// dynamics penalties' per-piece costs, one penalty after the other).  Shared by the host evaluation (svsdf_runtime.h: HostEval) and
// the device back end (svsdf_backend.cu).
struct BackendEvalView {
    MincoView m;
    double *times, *gradByTimes, *partialGradByTimes, *partialGradByCoeffs, *gradByPoints, *adj, *dynPartial;
};
// forwardT / forwardP (back_end_optimizer.hpp:353-354): tau -> T, MINCO, its energy (returned) and partial gradients
// (every lane returns the energy)
template <class Team = SerialTeam>
SVSDF_HD inline double backend_forward(const BackendEvalView &E, const double *x, const Team &team = Team()) {
    const int N = E.m.N;
    for (int i = team.lane(); i < N; i += team.size()) E.times[i] = forwardT(x[i]);
    team.sync();
    minco_set_parameters(E.m, x + N, E.times, team);
    const double energy = minco_energy(E.m);
    minco_energy_grad_coeffs(E.m, E.partialGradByCoeffs, team);
    minco_energy_grad_times(E.m, E.partialGradByTimes, team);
    team.sync();
    return energy;
}
// o: the device record [cost, gradC (18N), gradT (N), n_inside] of the trajectory backend_forward built; adds it, then the pose penalty
// when pose is not null (pose_rec: its sample records), then the dynamics penalty when dyn is not null (the reference's dyn_cost slot,
// back_end_optimizer.hpp:358, :387), propagates through MINCO and adds rho * sum(T).  Returns the cost (every lane), g the gradient
// w.r.t. x.  pos_out: the safety term and the pose penalty; other_out the rest.
template <class Team = SerialTeam>
SVSDF_HD inline double backend_backward(const BackendEvalView &E, double energy, const double *o, const double *x, double rho,
                                        const PoseParams *pose, const double *pose_rec, const DynamicsParams *dyn, double *g, double *pos_out,
                                        double *other_out, const Team &team = Team()) {
    const int N = E.m.N;
    double cost = energy;
    const double energy_cost = cost;
    cost += o[0];
    for (int e = team.lane(); e < 18 * N; e += team.size()) E.partialGradByCoeffs[e] += o[1 + e];
    for (int i = team.lane(); i < N; i += team.size()) E.partialGradByTimes[i] += o[1 + 18 * N + i];
    team.sync();
    if (pose) {
        cost += pose_penalty(*pose, N, E.times, E.m.b, pose_rec, E.partialGradByCoeffs, E.partialGradByTimes, E.dynPartial, team);
        team.sync();  // every lane has read the partials before the dynamics penalty rewrites them
    }
    const double pos_cost = cost - energy_cost;
    if (dyn) cost += dynamics_penalty(*dyn, N, E.times, E.m.b, E.partialGradByCoeffs, E.partialGradByTimes, E.dynPartial, team);
    minco_propagate(E.m, E.partialGradByCoeffs, E.partialGradByTimes, E.adj, E.gradByPoints, E.gradByTimes, team);
    double tsum = 0.0;
    for (int i = 0; i < N; ++i) tsum += E.times[i];
    cost += rho * tsum;
    for (int i = team.lane(); i < N; i += team.size()) E.gradByTimes[i] += rho;
    *pos_out = pos_cost;
    *other_out = cost - pos_cost;
    for (int i = team.lane(); i < N; i += team.size()) g[i] = backwardGradT(x[i], E.gradByTimes[i]);
    for (int i = team.lane(); i < 3 * (N - 1); i += team.size()) g[N + i] = E.gradByPoints[i];
    team.sync();
    return cost;
}

}  // namespace host
}  // namespace svsdf
