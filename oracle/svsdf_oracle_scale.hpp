// oracle/svsdf_oracle_scale.hpp — TEST INFRASTRUCTURE ONLY.
//
// The oracle's deformable-robot path: the reference with `#define useScale true` (sw_manager.hpp:17) and getScale(t)
// (:495-503) as this project's schedule S(t) = diag(a_x + sin(w_x t + phi_x) b_x, a_y + sin(w_y t + phi_y) b_y, 1).
// It extends the rigid restatement in svsdf_oracle.hpp (which it leaves as it is) with the scaled members; what the
// reference does with useScale on, and this file follows:
//   * choiceTInit's 2-argument overload (:538-581, called at :854) never reads its template flag: the seed scan stays
//     rigid (the inherited SweptVolume::choiceTInit);
//   * gradientDescent (:1249-1325), its FD slope (:798-806) and the FD gradient (:779-795) go through
//     getSDFAtTimeStamp<useScale> / getGradPrelAtTimeStamp<useScale>: rel = (Rt^T St^-1)(p - xt) (:528-535), the 3x3 product
//     formed first (eager Eigen), St at the sample's absolute time; the mesh functor's _igl variants zero xt(2) as before;
//   * St^-1 is Eigen 3.3's size-3 cofactor inverse: det = sy * sx, inv = 1/det, St^-1 = diag(sy inv, sx inv, (sx sy) inv);
//   * the interior branch (:916-1018) runs the scaled outer solve; its velocity fallback and ring do not change;
//   * the chain rule (back_end_optimizer.hpp:827, 1050) uses St = getScale(t*): sdf_grad = -L' (-(St^-1)^T rotate g); the
//     yaw term (:1062) has no St^-1 (exact only at St = I) and gdT no dS/dt term.
// tests/test_oracle_scale.py pins it bit for bit on the reference's own code built that way (`make -C oracle ref`).
#pragma once
#include "minco_oracle.hpp"
#include "svsdf_oracle.hpp"

namespace oracle {

struct ScaleSchedule {
    double a[2], b[2], w[2], phi[2];  // per axis x, y
};
// S(t) diagonal (sx, sy) and the diagonal of St.inverse()
inline void scale_at(const ScaleSchedule &z, double t, double s[2], double inv[3]) {
    double s0, c0, s1, c1;
    psc::sincos(z.w[0] * t + z.phi[0], s0, c0);
    psc::sincos(z.w[1] * t + z.phi[1], s1, c1);
    s[0] = z.a[0] + s0 * z.b[0];
    s[1] = z.a[1] + s1 * z.b[1];
    const double invdet = 1.0 / (s[1] * s[0]);
    inv[0] = s[1] * invdet;
    inv[1] = s[0] * invdet;
    inv[2] = (s[0] * s[1]) * invdet;
}

struct ScaledSweptVolume : SweptVolume {
    ScaleSchedule sched{};

    // getStateOnTrajStamp(t, xt, Rt, St) (:476-487) + posEva2Rel(p, xt, Rt, St) (:528-535)
    void relAtS(const double p[3], double t, double rel[3]) const {
        double xt[3];
        traj.getPos(t, xt);
        double s, c;
        psc::sincos(xt[2], s, c);
        if (shape.id == SH_MESH) xt[2] = 0;  // getSDFAtTimeStamp_igl<true> (:770-776)
        double sc[2], inv[3];
        scale_at(sched, t, sc, inv);
        double d0 = p[0] - xt[0], d1 = p[1] - xt[1], d2 = p[2] - xt[2];
        rel[0] = (c * inv[0]) * d0 + (s * inv[1]) * d1 + 0.0 * d2;
        rel[1] = (-s * inv[0]) * d0 + (c * inv[1]) * d1 + 0.0 * d2;
        rel[2] = 0.0 * d0 + 0.0 * d1 + inv[2] * d2;
    }
    double sdfAtS(const double p[3], double t) const {
        double rel[3];
        relAtS(p, t, rel);
        return shape_sdf(shape, rel[0], rel[1], rel[2]);
    }
    // getSDF_DOTAtTimeStamp<true> :798-806
    double sdfDotAtS(const double p[3], double t) const {
        double t1 = std::max(0.0, t - 0.000001);
        double t2 = std::min(traj_duration, t + 0.000001);
        return (sdfAtS(p, t2) - sdfAtS(p, t1)) * 500000;
    }
    // getGradPrelAtTimeStamp<true> :779-795
    void gradPrelAtS(const double p[3], double t, double g[3]) const {
        double rel[3];
        relAtS(p, t, rel);
        shape_grad1(shape, rel[0], rel[1], rel[2], g);
    }
    // gradientDescent :1249-1325 with getSDFAtTimeStamp<true>; f(x0) is evaluated on the scaled shape at iter == 0
    void gradientDescentS(double t_min, double t_max, const double x0, double &fx, double &x, const double p[3]) const {
        int max_iter = 1000;
        double alpha = 0.01, tau = alpha, g = 0.0, tol = 1e-16;
        x = x0;
        double change = 0;
        double prev_x = 10000000.0;
        int iter = 0;
        bool stop = false;
        double x_candidate, fx_candidate;
        while (iter < max_iter && !stop && std::abs(x - prev_x) > tol) {
            if (iter == 0) fx = sdfAtS(p, x);
            g = sdfDotAtS(p, x);
            tau = alpha;
            prev_x = x;
            for (int div = 1; div < 30; div++) {
                iter = iter + 1;
                g = sdfDotAtS(p, x);
                change = -tau * ((int)(g > 0) - (g < 0));
                x_candidate = x + change;
                x_candidate = std::max(std::min(x_candidate, t_max), t_min);
                fx_candidate = sdfAtS(p, x_candidate);
                if ((fx_candidate - fx) < 0) {
                    x = x_candidate;
                    fx = fx_candidate;
                    break;
                }
                tau = 0.5 * tau;
                if (div == 29) stop = true;
            }
        }
    }
    // getSDFofSweptVolume<false,true> :844-866 (choiceTInit rigid)
    double getSDFofSweptVolumeS(const double p[3], double &time_seed_f, double grad_prel[3]) const {
        double t_star = 0.0, sdf_star = 0.0;
        double ts = choiceTInit(p, 0.15);
        double tmin_ = std::max(0.0, ts - 3.4);
        double tmax_ = std::min(ts + 3.4, traj_duration);
        gradientDescentS(tmin_, tmax_, ts, sdf_star, t_star, p);
        gradPrelAtS(p, t_star, grad_prel);
        time_seed_f = t_star;
        return sdf_star;
    }
    // getTrueSDFofSweptVolume<true> :916-1018 (same control flow as SweptVolume::getTrueSDFofSweptVolume)
    double getTrueSDFofSweptVolumeS(const double p[3], double &time_seed_f, double grad_prel[3], int *gsip_rounds = nullptr) const {
        const double PI = 3.14159265358979323846;
        if (gsip_rounds) *gsip_rounds = 0;
        double argmin_dis = getSDFofSweptVolumeS(p, time_seed_f, grad_prel);
        if (argmin_dis > 0) return argmin_dis;
        double vel[3];
        traj.getVel(time_seed_f, vel);
        auto norm3 = [](const double v[3]) { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); };
        if (norm3(vel) < 0.01) {
            if (time_seed_f < 0.1) {
                for (double t_scan = time_seed_f; t_scan <= traj_duration; t_scan += 0.1) {
                    traj.getVel(t_scan, vel);
                    if (norm3(vel) >= 0.01) break;
                }
            } else if (time_seed_f > traj_duration - 0.1) {
                for (double t_scan = time_seed_f; t_scan >= 0; t_scan -= 0.1) {
                    traj.getVel(t_scan, vel);
                    if (norm3(vel) >= 0.01) break;
                }
            }
        }
        double cx = p[0], cy = p[1];
        double r = 10;
        double theta0 = psc::atan2(vel[0], -vel[1]);
        if (theta0 < 0) theta0 += 2 * PI;
        double theta_res = PI + 0.1;
        const double rk_res = 1.5, rk0 = 1.0;
        double r_star = 0, max_g, cur_g, real_t_star = 0, star_rk = 0, star_theta = 0;
        int iter = 1;
        double yk3[3], gtmp[3];
        while (true) {
            max_g = -100000;
            for (double rk = rk0; rk > 0; rk -= rk_res) {
                for (double theta = theta0; theta < theta0 + 2 * PI; theta += theta_res) {
                    double sth, cth;
                    psc::sincos(theta, sth, cth);
                    yk3[0] = cx + rk * r * cth;
                    yk3[1] = cy + rk * r * sth;
                    yk3[2] = 0.0;
                    cur_g = getSDFofSweptVolumeS(yk3, time_seed_f, gtmp);
                    if (cur_g > max_g) {
                        max_g = cur_g;
                        real_t_star = time_seed_f;
                        star_rk = rk;
                        star_theta = theta;
                    }
                }
            }
            r_star = r - max_g;
            r = r_star;
            if (gsip_rounds) (*gsip_rounds)++;
            if (iter > 8) break;
            if (std::abs(max_g) < 0.1) break;
            theta_res /= (2 + 1);
            theta_res = std::max(0.3, theta_res);
            theta0 = star_theta;
            iter++;
        }
        double sst, cst;
        psc::sincos(star_theta, sst, cst);
        double corx = cx + star_rk * r_star * cst;
        double cory = cy + star_rk * r_star * sst;
        double gx = corx - p[0], gy = cory - p[1], gz = 0.0;
        double z = gx * gx + gy * gy + gz * gz;
        if (z > 0) {
            double n = std::sqrt(z);
            gx /= n; gy /= n; gz /= n;
        }
        grad_prel[0] = gx; grad_prel[1] = gy; grad_prel[2] = gz;
        time_seed_f = real_t_star;
        return -r_star;
    }
};

// addSaftyPenaOnSweptVolumeParallelTrueSDF :774-869 + grad_cost_p_sw :1031-1066 with St = getScale(t*)
inline void addSafetyPenaltyTrueSDFScaled(const ScaledSweptVolume &sv, const CostParams &cp, int N, const double *coeffs,
                                          const double *points, int64_t P, int stride, double &cost, double *gradT, double *gradC,
                                          PointResult *per_point, int64_t *n_inside = nullptr) {
    const double weightPos = cp.weight_p;
    int64_t inside = 0;
#pragma omp parallel for num_threads(cp.threads) schedule(dynamic) reduction(+ : inside)
    for (int64_t k = 0; k < P; ++k) {
        double pos_eva[3] = {points[k * stride], points[k * stride + 1], 0.0};
        double gradp_rel[3] = {0, 0, 0};
        double time_star = 0.0;
        double sdf_value = sv.getTrueSDFofSweptVolumeS(pos_eva, time_star, gradp_rel);
        if (!(sdf_value > 0)) inside++;
        double time_local = time_star;
        int i = sv.traj.locatePieceIdx(time_local);
        double s1 = time_local, s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2, s5 = s4 * s1;
        double beta0[6] = {1.0, s1, s2, s3, s4, s5};
        double beta1[6] = {0.0, 1.0, 2.0 * s1, 3.0 * s2, 4.0 * s3, 5.0 * s4};
        double pos[3], vel[3];
        for (int d = 0; d < 3; ++d) {
            const double *c = coeffs + d * 6 * N + 6 * i;
            double a = 0, b = 0;
            for (int q = 0; q < 6; ++q) { a += c[q] * beta0[q]; b += c[q] * beta1[q]; }
            pos[d] = a; vel[d] = b;
        }
        double yaw = pos[2];
        double sy, cy;
        psc::sincos(yaw, sy, cy);
        pos[2] = 0.0;
        if (sdf_value < 0) {
            double g0 = cy * gradp_rel[0] + sy * gradp_rel[1];
            double g1 = -sy * gradp_rel[0] + cy * gradp_rel[1];
            gradp_rel[0] = g0; gradp_rel[1] = g1;
        }
        double sc[2], inv[3];
        scale_at(sv.sched, time_star, sc, inv);
        const double ix = inv[0], iy = inv[1];
        double sdf_cost = -1.0, sdf_out_grad = 0.0;
        smoothedL1(cp.safety_hor - sdf_value, 0.01, sdf_cost, sdf_out_grad);
        // sdf_grad = -L' * ( -(St^-1)^T * rotate * g )
        double rg0 = -((ix * cy) * gradp_rel[0] + (-(ix * sy)) * gradp_rel[1]);
        double rg1 = -((iy * sy) * gradp_rel[0] + (iy * cy) * gradp_rel[1]);
        double sdf_grad0 = -sdf_out_grad * rg0, sdf_grad1 = -sdf_out_grad * rg1;
        double costp = 0.0, gradp[2] = {0, 0}, grad_yaw_v = 0.0;
        bool active = false;
        if (sdf_cost > 0) {
            costp += sdf_cost;
            gradp[0] += sdf_grad0;
            gradp[1] += sdf_grad1;
            double d0 = pos_eva[0] - pos[0], d1 = pos_eva[1] - pos[1];
            double w0 = -sy * d0 + cy * d1;
            double w1 = -cy * d0 + -sy * d1;
            grad_yaw_v = (-sdf_out_grad * gradp_rel[0]) * w0 + (-sdf_out_grad * gradp_rel[1]) * w1;  // no St^-1 (:1062)
            active = costp > 0;
        }
        double G[3] = {0, 0, 0}, pena = 0.0;
        if (active) {  // accumulated from zero as the rigid loop does (signed zeros included)
            G[0] += weightPos * gradp[0];
            G[1] += weightPos * gradp[1];
            G[2] += weightPos * grad_yaw_v;
            pena += weightPos * costp;
        }
        double gdT = -(G[0] * vel[0] + G[1] * vel[1] + G[2] * vel[2]);
        if (per_point) {
            PointResult &pr = per_point[k];
            pr.sdf = sdf_value; pr.tstar = time_star;
            pr.g[0] = gradp_rel[0]; pr.g[1] = gradp_rel[1]; pr.g[2] = gradp_rel[2];
            pr.piece = i; pr.pena = pena;
        }
#pragma omp critical
        {
            cost += pena;
            for (int d = 0; d < 3; ++d)
                for (int q = 0; q < 6; ++q) gradC[d * 6 * N + 6 * i + q] += beta0[q] * G[d];
            for (int j = 0; j < i; ++j) gradT[j] += gdT;
        }
    }
    if (n_inside) *n_inside = inside;
}

}  // namespace oracle
