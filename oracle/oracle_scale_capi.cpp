// oracle/oracle_scale_capi.cpp — TEST INFRASTRUCTURE ONLY: C entry points (for ctypes, oracle/scale_py.py) over the
// oracle's deformable-robot path (svsdf_oracle_scale.hpp).  Built by oracle/Makefile into _build/libsvsdf_oracle_scale.so
// (portable sin/cos: the strict CUDA build's bits) and _build/libsvsdf_oracle_scale_glibc.so (glibc sin/cos).
#include <omp.h>

#include <cstring>
#include <vector>

#include "svsdf_oracle_scale.hpp"

using namespace oracle;

namespace {
struct ScaledOracle {
    ScaledSweptVolume sv;
    CostParams cp;
    std::vector<double> points;  // stride 3
    int64_t P = 0;
};
ScaleSchedule unpack(const double *s) {  // a_x, a_y, b_x, b_y, w_x, w_y, phi_x, phi_y
    ScaleSchedule z;
    for (int d = 0; d < 2; ++d) { z.a[d] = s[d]; z.b[d] = s[2 + d]; z.w[d] = s[4 + d]; z.phi[d] = s[6 + d]; }
    return z;
}
ScaledOracle *make(Shape S, double weight_p, double safety_hor, int threads) {
    ScaledOracle *o = new ScaledOracle();
    o->sv.shape = S;
    o->cp.weight_p = weight_p;
    o->cp.safety_hor = safety_hor;
    o->cp.threads = threads > 0 ? threads : 1;
    return o;
}
}  // namespace

extern "C" {

void *sorc_create(const char *name, const double *poly_params, const double *poly_xy, int poly_n, double weight_p,
                  double safety_hor, int threads) {
    Shape S;  // the registry lookup of oracle_capi.cpp's make_shape
    S.id = shape_id_from_name(name ? name : "");
    if (poly_params) S.set_poly_params(poly_params[0], poly_params[1], poly_params[2]);
    if (S.id == SH_POLYGON) {
        if (poly_xy && poly_n >= 3) S.set_polygon(poly_xy, poly_n);
        else S.set_default_rect();
    }
    return make(S, weight_p, safety_hor, threads);
}
void *sorc_create_mesh(const double *poly_params, const double *V, int nv, const int *F, int nf, double weight_p,
                       double safety_hor, int threads) {
    Shape S;
    S.id = SH_MESH;
    if (poly_params) S.set_poly_params(poly_params[0], poly_params[1], poly_params[2]);
    S.set_mesh(V, nv, F, nf);
    return make(S, weight_p, safety_hor, threads);
}
void sorc_destroy(void *h) { delete (ScaledOracle *)h; }
void sorc_set_threads(void *h, int threads) { ((ScaledOracle *)h)->cp.threads = threads > 0 ? threads : 1; }
void sorc_set_scale(void *h, const double *sched) { ((ScaledOracle *)h)->sv.sched = unpack(sched); }
void sorc_scale_at(const double *sched, double t, double *s2, double *inv3) { scale_at(unpack(sched), t, s2, inv3); }
void sorc_set_points(void *h, const double *pts, int64_t P, int stride) {
    ScaledOracle *o = (ScaledOracle *)h;
    o->points.resize((size_t)P * 3);
    for (int64_t i = 0; i < P; ++i) {
        o->points[3 * i] = pts[i * stride];
        o->points[3 * i + 1] = pts[i * stride + 1];
        o->points[3 * i + 2] = stride > 2 ? pts[i * stride + 2] : 0.0;
    }
    o->P = P;
}
void sorc_set_traj(void *h, int N, const double *T, const double *coeffs) {
    Trajectory tr;
    trajectory_from_coeffs(N, T, coeffs, tr);
    ((ScaledOracle *)h)->sv.updateTraj(tr);
}
double sorc_duration(void *h) { return ((ScaledOracle *)h)->sv.traj_duration; }
void sorc_traj_pos(void *h, double t, double *p3) { ((ScaledOracle *)h)->sv.traj.getPos(t, p3); }
void sorc_traj_vel(void *h, double t, double *v3) { ((ScaledOracle *)h)->sv.traj.getVel(t, v3); }
// getSDFAtTimeStamp at one absolute time t: scaled != 0 the descent's getSDFAtTimeStamp<true>, scaled == 0 the rigid one of
// the seed scan (choiceTInit stays rigid)
double sorc_sdf_at(void *h, const double *p3, double t, int scaled) {
    const ScaledSweptVolume &sv = ((ScaledOracle *)h)->sv;
    return scaled ? sv.sdfAtS(p3, t) : sv.sdfAt(p3, t);
}
void sorc_gradient_descent(void *h, const double *p3, double tmin, double tmax, double x0, double *fx, double *x) {
    ((ScaledOracle *)h)->sv.gradientDescentS(tmin, tmax, x0, *fx, *x, p3);
}
// getSDFofSweptVolume<false,true> per point: the outer solve alone (body-frame gradient); pts stride 3
void sorc_query_outer(void *h, int64_t P, const double *pts, double *sdf, double *tstar, double *grad3) {
    ScaledOracle *o = (ScaledOracle *)h;
#pragma omp parallel for num_threads(o->cp.threads) schedule(dynamic)
    for (int64_t i = 0; i < P; ++i) {
        double p[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
        double g[3], ts = 0;
        sdf[i] = o->sv.getSDFofSweptVolumeS(p, ts, g);
        tstar[i] = ts;
        grad3[3 * i] = g[0]; grad3[3 * i + 1] = g[1]; grad3[3 * i + 2] = g[2];
    }
}
// getTrueSDFofSweptVolume<true> per point (world-frame direction for sdf <= 0); pts stride 3
void sorc_query(void *h, int64_t P, const double *pts, double *sdf, double *tstar, double *grad3, int *rounds) {
    ScaledOracle *o = (ScaledOracle *)h;
#pragma omp parallel for num_threads(o->cp.threads) schedule(dynamic)
    for (int64_t i = 0; i < P; ++i) {
        double p[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
        double g[3], ts = 0;
        int r = 0;
        sdf[i] = o->sv.getTrueSDFofSweptVolumeS(p, ts, g, &r);
        tstar[i] = ts;
        grad3[3 * i] = g[0]; grad3[3 * i + 1] = g[1]; grad3[3 * i + 2] = g[2];
        if (rounds) rounds[i] = r;
    }
}
// the penalty loop (accumulating); per_point: P x 7 (sdf, tstar, gx, gy, gz, piece, pena) or NULL; returns n_inside
int64_t sorc_cost_grad(void *h, int N, const double *T, const double *coeffs, double *cost_io, double *gradT_io, double *gradC_io,
                       double *per_point) {
    ScaledOracle *o = (ScaledOracle *)h;
    sorc_set_traj(h, N, T, coeffs);
    std::vector<PointResult> pr;
    if (per_point) pr.resize(o->P);
    int64_t inside = 0;
    addSafetyPenaltyTrueSDFScaled(o->sv, o->cp, N, coeffs, o->points.data(), o->P, 3, *cost_io, gradT_io, gradC_io,
                                  per_point ? pr.data() : nullptr, &inside);
    if (per_point)
        for (int64_t i = 0; i < o->P; ++i) {
            double *r = per_point + 7 * i;
            r[0] = pr[i].sdf; r[1] = pr[i].tstar; r[2] = pr[i].g[0]; r[3] = pr[i].g[1]; r[4] = pr[i].g[2];
            r[5] = pr[i].piece; r[6] = pr[i].pena;
        }
    return inside;
}

}  // extern "C"
