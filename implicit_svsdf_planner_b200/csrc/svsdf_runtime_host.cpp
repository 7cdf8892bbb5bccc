// svsdf_runtime_host.cpp — the entry points that need no context: mesh reading and its winding numbers, the LMBM plug-in, the mid
// end, MINCO and the tau map, the dynamics penalty and the scale matrix, all on the host.
#include <dlfcn.h>
#include <unistd.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "host/fwn_bvh.hpp"
#include "host/mid_end.hpp"
#include "svsdf_runtime.h"

namespace {

// The fdlibm sin of csrc/svsdf_sincos.cuh (Cody–Waite reduction, k_sin.c / k_cos.c polynomials with FMA) on the host,
// for |x| < 1e6 (svsdf_set_scale keeps the schedule's arguments there): svsdf_scale_matrix returns the kernels' bits.
double sin_portable_host(double x) {
    const double v = std::fma(x, 0x1.45f306dc9c883p-1, 6755399441055744.0);
    int64_t vb;
    std::memcpy(&vb, &v, sizeof(vb));
    const int q = (int)(uint32_t)(vb & 0xffffffffLL);
    const double fn = v - 6755399441055744.0;
    double r = std::fma(fn, -0x1.921fb54442d18p+0, x);
    r = std::fma(fn, -0x1.1a62633145c07p-54, r);
    r = std::fma(fn, 0x1.f1976b7ed8fbcp-110, r);
    const double z = r * r;
    double ps = std::fma(z, 1.58969099521155010221e-10, -2.50507602534068634195e-08);
    ps = std::fma(z, ps, 2.75573137070700676789e-06);
    ps = std::fma(z, ps, -1.98412698298579493134e-04);
    ps = std::fma(z, ps, 8.33333333332248946124e-03);
    ps = std::fma(z, ps, -1.66666666666666324348e-01);
    const double sr = std::fma(r * z, ps, r);
    double pc = std::fma(z, -1.13596475577881948265e-11, 2.08757232129817482790e-09);
    pc = std::fma(z, pc, -2.75573143513906633035e-07);
    pc = std::fma(z, pc, 2.48015872894767294178e-05);
    pc = std::fma(z, pc, -1.38888888888741095749e-03);
    pc = std::fma(z, pc, 4.16666666666666019037e-02);
    const double cr = std::fma(z * z, pc, std::fma(z, -0.5, 1.0));
    const double ss = (q & 1) ? cr : sr;
    return (q & 2) ? -ss : ss;
}

}  // namespace

extern "C" {

// Wavefront .obj -> (V, F): `v x y z` and `f i[/..] j[/..] k[/..] ...` records (1-based or negative indices), polygons
// fan-triangulated — what igl::read_triangle_mesh yields for the reference's shapes/*.obj (Shape.hpp:285).
int svsdf_read_obj(const char *path, double **vertices_out, int *nv_out, int32_t **faces_out, int *nf_out) {
    if (!path || !vertices_out || !nv_out || !faces_out || !nf_out) return SVSDF_ERR_INVALID;
    *vertices_out = nullptr; *faces_out = nullptr; *nv_out = 0; *nf_out = 0;
    std::FILE *fp = std::fopen(path, "r");
    if (!fp) return SVSDF_ERR_INVALID;
    std::vector<double> V;
    std::vector<int32_t> F;
    char line[4096];
    bool bad = false;
    while (std::fgets(line, sizeof(line), fp)) {
        const size_t len = std::strlen(line);
        if (len + 1 == sizeof(line) && line[len - 1] != '\n') { bad = true; break; }  // record longer than the buffer
        char *p = line;
        while (*p == ' ' || *p == '\t') ++p;
        if (p[0] == 'v' && (p[1] == ' ' || p[1] == '\t')) {
            double x, y, z;
            if (std::sscanf(p + 1, "%lf %lf %lf", &x, &y, &z) != 3) { bad = true; break; }
            V.push_back(x); V.push_back(y); V.push_back(z);
        } else if (p[0] == 'f' && (p[1] == ' ' || p[1] == '\t')) {
            std::vector<int32_t> idx;
            char *q = p + 1;
            for (;;) {
                while (*q == ' ' || *q == '\t') ++q;
                if (*q == 0 || *q == '\n' || *q == '\r' || *q == '#') break;
                char *end = nullptr;
                long i = std::strtol(q, &end, 10);
                if (end == q) { bad = true; break; }
                const long nv = (long)(V.size() / 3);
                idx.push_back((int32_t)(i > 0 ? i - 1 : nv + i));
                q = end;
                while (*q && *q != ' ' && *q != '\t' && *q != '\n' && *q != '\r') ++q;  // skip /vt/vn
            }
            if (bad) break;
            for (size_t k = 1; k + 1 < idx.size(); ++k) { F.push_back(idx[0]); F.push_back(idx[k]); F.push_back(idx[k + 1]); }
        }
    }
    std::fclose(fp);
    const int nv = (int)(V.size() / 3), nf = (int)(F.size() / 3);
    for (int32_t i : F)
        if (i < 0 || i >= nv) bad = true;
    if (bad || nv == 0 || nf == 0) return SVSDF_ERR_INVALID;
    double *vo = (double *)std::malloc(V.size() * sizeof(double));
    int32_t *fo = (int32_t *)std::malloc(F.size() * sizeof(int32_t));
    if (!vo || !fo) { std::free(vo); std::free(fo); return SVSDF_ERR_INVALID; }
    std::memcpy(vo, V.data(), V.size() * sizeof(double));
    std::memcpy(fo, F.data(), F.size() * sizeof(int32_t));
    *vertices_out = vo; *faces_out = fo; *nv_out = nv; *nf_out = nf;
    return SVSDF_OK;
}
int svsdf_mesh_fwn_host(const double *vertices, int nv, const int32_t *faces, int nf, int *n_nodes_out, int node_capacity,
                        uint32_t *children_out, float *data_out, int64_t n, const double *q, double *w_out) {
    if (!vertices || !faces || nv < 3 || nf < 1 || n < 0 || (n > 0 && (!q || !w_out))) return SVSDF_ERR_INVALID;
    for (int64_t k = 0; k < 3 * (int64_t)nf; ++k)
        if (faces[k] < 0 || faces[k] >= nv) return SVSDF_ERR_INVALID;
    host::FwnBvh B;
    B.build(vertices, nv, faces, nf);
    if (n_nodes_out) *n_nodes_out = B.nn;
    if (children_out && node_capacity >= B.nn) std::memcpy(children_out, B.child.data(), B.child.size() * sizeof(uint32_t));
    if (data_out && node_capacity >= B.nn) std::memcpy(data_out, B.data.data(), B.data.size() * sizeof(float));
    for (int64_t i = 0; i < n; ++i) w_out[i] = B.winding_number(q + 3 * i);
    return SVSDF_OK;
}

void svsdf_free(void *p) { std::free(p); }

// ---------------------------------------------------------------------------------------------------------------------
// The reference's LMBM library as a plug-in (lmbm.h:214-221).  Each handle is its own dlopen of (a private copy of) the file.
// ---------------------------------------------------------------------------------------------------------------------
static thread_local std::string g_lmbm_err;
const char *svsdf_lmbm_last_error(void) { return g_lmbm_err.c_str(); }
void svsdf_lmbm_default_params(svsdf_lmbm_params *p) {  // the member initialisers of lmbm::lmbm_parameter_t (lmbm.h:15-174)
    if (!p) return;
    p->timeout = 300.0f; p->bundle_size = 2; p->ini_corrections = 7; p->max_corrections = 15; p->exponent_distmeasure = 2;
    p->max_iterations = 10000; p->max_evaluations = 20000; p->past = 10; p->verbose = -1; p->update_method = 0; p->scaling_strategy = 0;
    p->delta_past = 1.0e-8; p->f_rel_eps = 1.0e+4; p->f_lower_bound = -1.0e+60; p->terminate_param1 = 1.0e-6; p->terminate_param2 = 1.0e-6;
    p->distance_measure = 0.5; p->sufficient_dec = 1.0e-4; p->max_stepsize = 1.5;
}
int svsdf_lmbm_open(const char *path, int private_copy, svsdf_lmbm **out) {
    if (!path || !out) return SVSDF_ERR_INVALID;
    *out = nullptr;
    std::string load = path;
    bool temp = false;
    if (private_copy) {  // a distinct file is a distinct library instance to the loader: own statics, own Fortran COMMON / SAVE data
        FILE *src = std::fopen(path, "rb");
        if (!src) { g_lmbm_err = std::string("svsdf_lmbm_open: cannot read ") + path; return SVSDF_ERR_INVALID; }
        char tmpl[] = "/tmp/svsdf_lmbm_XXXXXX";
        const int fd = mkstemp(tmpl);
        if (fd < 0) { std::fclose(src); g_lmbm_err = "svsdf_lmbm_open: mkstemp failed"; return SVSDF_ERR_INVALID; }
        char buf[1 << 16];
        size_t nrd;
        bool ok = true;
        while ((nrd = std::fread(buf, 1, sizeof(buf), src)) > 0) ok = ok && (write(fd, buf, nrd) == (ssize_t)nrd);
        std::fclose(src);
        close(fd);
        if (!ok) { unlink(tmpl); g_lmbm_err = "svsdf_lmbm_open: copy failed"; return SVSDF_ERR_INVALID; }
        load = tmpl;
        temp = true;
    }
    void *dl = dlopen(load.c_str(), RTLD_NOW | RTLD_LOCAL);
    if (temp) unlink(load.c_str());  // the mapping stays valid
    if (!dl) { g_lmbm_err = std::string("svsdf_lmbm_open: dlopen: ") + (dlerror() ? dlerror() : "?"); return SVSDF_ERR_INVALID; }
    void *sym = dlsym(dl, "_ZN4lmbm13lmbm_optimizeEiPdS0_PFdPvPKdS0_iES1_PFiS1_S3_iEPNS_16lmbm_parameter_tE");
    if (!sym) { dlclose(dl); g_lmbm_err = "svsdf_lmbm_open: lmbm::lmbm_optimize not found in the library"; return SVSDF_ERR_INVALID; }
    svsdf_lmbm *h = new svsdf_lmbm();
    h->dl = dl;
    h->optimize = reinterpret_cast<decltype(h->optimize)>(sym);
    *out = h;
    return SVSDF_OK;
}
void svsdf_lmbm_close(svsdf_lmbm *h) {
    if (!h) return;
    if (h->dl) dlclose(h->dl);
    delete h;
}
int svsdf_lmbm_minimize(svsdf_lmbm *h, svsdf_eval_t eval, void *instance, double *x, int n, const svsdf_lmbm_params *params,
                        svsdf_progress_t progress, double *f_out) {
    if (!h || !h->optimize || !eval || !x || n < 1) return SVSDF_ERR_INVALID;
    svsdf_lmbm_params p;
    if (params) p = *params; else svsdf_lmbm_default_params(&p);
    double fx = 0.0;
    // lmbm.cpp calls the progress function unconditionally (earlyexit_): never hand it a null pointer
    const int ret = h->optimize(n, x, &fx, eval, instance, progress ? progress : +[](void *, const double *, const int) { return 0; }, &p);
    if (f_out) *f_out = fx;
    return ret;
}

// ---------------------------------------------------------------------------------------------------------------------
// mid end (host/mid_end.hpp): OriTraj's cost function and warm-start optimisation, host only
// ---------------------------------------------------------------------------------------------------------------------
void svsdf_mid_default_config(svsdf_mid_config *c) {
    if (!c) return;
    const host::MidEndConfig d;
    c->rho_mid_end = d.rho_mid_end; c->vmax = d.vmax; c->omgmax = d.omgmax; c->weight_v = d.weight_v; c->weight_omg = d.weight_omg;
    c->weight_pr = d.weight_pr; c->weight_ar = d.weight_ar; c->smoothingEps = d.smoothingEps; c->integralIntervs = d.integralIntervs;
    c->vehicleMass = d.vehicleMass; c->gravAcc = d.gravAcc; c->horizDrag = d.horizDrag; c->vertDrag = d.vertDrag; c->parasDrag = d.parasDrag;
    c->speedEps = d.speedEps; c->mem_size = d.mem_size; c->past = d.past; c->min_step = d.min_step; c->g_epsilon = d.g_epsilon;
    c->relCostTolMidEnd = d.relCostTolMidEnd; c->max_iterations = d.max_iterations; c->cancel_after = d.cancel_after; c->solver = d.solver;
}
static host::MidEndConfig mid_cfg(const svsdf_mid_config *c) {
    host::MidEndConfig d;
    if (!c) return d;
    d.rho_mid_end = c->rho_mid_end; d.vmax = c->vmax; d.omgmax = c->omgmax; d.weight_v = c->weight_v; d.weight_omg = c->weight_omg;
    d.weight_pr = c->weight_pr; d.weight_ar = c->weight_ar; d.smoothingEps = c->smoothingEps; d.integralIntervs = c->integralIntervs;
    d.vehicleMass = c->vehicleMass; d.gravAcc = c->gravAcc; d.horizDrag = c->horizDrag; d.vertDrag = c->vertDrag; d.parasDrag = c->parasDrag;
    d.speedEps = c->speedEps; d.mem_size = c->mem_size; d.past = c->past; d.min_step = c->min_step; d.g_epsilon = c->g_epsilon;
    d.relCostTolMidEnd = c->relCostTolMidEnd; d.max_iterations = c->max_iterations; d.cancel_after = c->cancel_after; d.solver = c->solver;
    return d;
}
static bool mid_args_ok(const svsdf_mid_config *c, int N, const double *initS, const double *finalS, const double *Q, const double *rot) {
    return N >= 2 && N <= kMaxPieces && initS && finalS && Q && rot && (!c || (c->integralIntervs >= 1 && c->smoothingEps > 0.0 && c->vehicleMass > 0.0));
}
int svsdf_mid_cost(const svsdf_mid_config *cfg, int N, const double *initS, const double *finalS, const double *Q, const double *rot_list,
                   const double *x, double *cost_out, double *grad_out) {
    if (!mid_args_ok(cfg, N, initS, finalS, Q, rot_list) || !x || !cost_out || !grad_out) return SVSDF_ERR_INVALID;
    host::MidEnd M(mid_cfg(cfg));
    M.setup(initS, finalS, N, Q, rot_list);
    *cost_out = M.cost(x, grad_out);
    return SVSDF_OK;
}
int svsdf_mid_get_ori_traj(const svsdf_mid_config *cfg, int N, const double *initS, const double *finalS, const double *Q,
                           const double *T_init, const double *rot_list, double *opt_x_out, double *T_out, double *coeffs_out,
                           double *final_cost_out, int *iterations_out) {
    if (!mid_args_ok(cfg, N, initS, finalS, Q, rot_list) || !T_init || !opt_x_out) return SVSDF_ERR_INVALID;
    for (int i = 0; i < N; ++i)
        if (!(T_init[i] > 0.0)) return SVSDF_ERR_INVALID;
    host::MidEnd M(mid_cfg(cfg));
    M.setup(initS, finalS, N, Q, rot_list);
    return M.optimize(T_init, opt_x_out, T_out, coeffs_out, final_cost_out, iterations_out);
}

int svsdf_minco_forward(const double *initS, const double *finalS, int N, const double *q, const double *T,
                        double *coeffs_out, double *energy, double *gradC_out, double *gradT_out) {
    if (!initS || !finalS || !q || !T || N < 2) return SVSDF_ERR_INVALID;
    host::MincoS3NU m;
    m.setConditions(initS, finalS, N);
    m.setParameters(q, T);
    if (coeffs_out) std::memcpy(coeffs_out, m.getCoeffs(), sizeof(double) * 18 * N);
    if (energy) *energy = m.getEnergy();
    if (gradC_out) m.getEnergyPartialGradByCoeffs(gradC_out);
    if (gradT_out) m.getEnergyPartialGradByTimes(gradT_out);
    return SVSDF_OK;
}

int svsdf_minco_propagate(const double *initS, const double *finalS, int N, const double *q, const double *T,
                          const double *gradC, const double *gradT, double *gradQ_out, double *gradT_out) {
    if (!initS || !finalS || !q || !T || !gradC || !gradT || !gradQ_out || !gradT_out || N < 2) return SVSDF_ERR_INVALID;
    host::MincoS3NU m;
    m.setConditions(initS, finalS, N);
    m.setParameters(q, T);
    m.propogateGrad(gradC, gradT, gradQ_out, gradT_out);
    return SVSDF_OK;
}

void svsdf_forward_T(int n, const double *tau, double *T) { for (int i = 0; i < n; ++i) T[i] = host::forwardT(tau[i]); }
void svsdf_backward_T(int n, const double *T, double *tau) { for (int i = 0; i < n; ++i) tau[i] = host::backwardT(T[i]); }

void svsdf_default_dynamics(svsdf_dynamics *dyn) {
    if (!dyn) return;
    dyn->vmax = 10.0; dyn->omgmax = 10.0; dyn->weight_v = 10.0; dyn->weight_omg = 10.0; dyn->smoothingEps = 1.0e-2;
    dyn->integralIntervs = 4;
}

int svsdf_dynamics_penalty(const svsdf_dynamics *dyn, int N, const double *T, const double *coeffs, double *cost, double *gradC,
                           double *gradT) {
    if (!dyn || !dynamics_valid(*dyn) || N < 1 || !T || !coeffs || !cost || !gradC || !gradT) return SVSDF_ERR_INVALID;
    std::vector<double> gc((size_t)18 * N, 0.0), gt(N, 0.0), partial(N, 0.0);
    const double c = host::dynamics_penalty(to_host_dynamics(*dyn), N, T, coeffs, gc.data(), gt.data(), partial.data());
    *cost = c;
    std::memcpy(gradC, gc.data(), sizeof(double) * 18 * N);
    std::memcpy(gradT, gt.data(), sizeof(double) * N);
    return SVSDF_OK;
}

void svsdf_default_pose_penalty(svsdf_pose_penalty *p) {
    if (!p) return;
    p->weight = 60.0;  // weight_p
    p->integralIntervs = 4;
    p->half[0] = p->half[1] = p->half[2] = 8.5;  // kernel_size * occupancy_resolution / 2 = 17 * 1.0 / 2
}

int svsdf_scale_matrix(const svsdf_scale *scale, double t, double S_out[9], double Sinv_out[9]) {
    if (!scale || !scale_valid(*scale) || !std::isfinite(t)) return SVSDF_ERR_INVALID;
    // the arithmetic of scale_inv (svsdf_kernels.cuh) and Eigen 3.3's size-3 inverse of diag(sx, sy, 1)
    const double sx = scale->a[0] + sin_portable_host(scale->w[0] * t + scale->phi[0]) * scale->b[0];
    const double sy = scale->a[1] + sin_portable_host(scale->w[1] * t + scale->phi[1]) * scale->b[1];
    const double inv = 1.0 / (sy * sx);
    if (S_out) {
        for (int k = 0; k < 9; ++k) S_out[k] = 0.0;
        S_out[0] = sx; S_out[4] = sy; S_out[8] = 1.0;
    }
    if (Sinv_out) {
        for (int k = 0; k < 9; ++k) Sinv_out[k] = 0.0;
        Sinv_out[0] = sy * inv; Sinv_out[4] = sx * inv; Sinv_out[8] = (sx * sy) * inv;
    }
    return SVSDF_OK;
}

}  // extern "C"
