// svsdf_runtime_context.cpp — a context's life (svsdf_create / svsdf_destroy), its shape, query points and settings, and the
// kernel-variant table; the small per-context entry points (counters, sincos and shape evaluation).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <limits>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "host/fwn_bvh.hpp"
#include "svsdf_runtime.h"

#define SVSDF_VARIANT(NS, SCALED)                                                                                      \
    {NS##SCALED::query_occupancy,  NS##SCALED::launch_cost_kernels, NS::launch_pose_table,                            \
     NS::launch_finalize,          NS::launch_shape_eval,           NS::launch_sincos,                                \
     NS##_multi##SCALED::launch_multi, NS##_multi::launch_pose_multi, NS##_multi::launch_compact_multi,              \
     NS##_multi::launch_finalize_multi, NS::launch_pose}
const Kernels kKernels[2][2] = {{SVSDF_VARIANT(fast, ), SVSDF_VARIANT(fast, _scaled)}, {SVSDF_VARIANT(strict, ), SVSDF_VARIANT(strict, _scaled)}};
#undef SVSDF_VARIANT

namespace {

const char *kShapeNames[] = {"star",      "sdHorseshoe", "sdPie",      "sdPie2", "sdArc",          "sdTunnel",
                             "sdCutDisk", "sdTrapezoid", "sdRhombus",  "sdHeart", "sdRoundedX",    "bigX",
                             "sdRoundedCross", "sdOrientedVesica", "sdMoon", "sdUnevenCapsule"};

int shape_id_from_name(const char *name) {
    if (name) {
        for (int i = 0; i < 16; ++i)
            if (std::strcmp(name, kShapeNames[i]) == 0) return i;
        if (std::strcmp(name, "Circle") == 0) return SH_CIRCLE;
    }
    return SH_POLYGON;  // sw_manager.hpp:363-372
}

// Host-side construction of the shape functor parameters (what the reference's shape constructors do:
// Shape.hpp:281-294 base transform, and the per-class constant members).
void build_shape(const svsdf_config &cfg, ShapeParams &S) {
    std::memset(&S, 0, sizeof(S));
    S.id = shape_id_from_name(cfg.shape);
    const double PI = 3.14159265358979323846;  // Shape.hpp:31
    const double yaw = (cfg.poly_params[2] * PI / 180.0);
    S.trans[0] = cfg.poly_params[0];
    S.trans[1] = cfg.poly_params[1];
    S.rot[0] = std::cos(yaw);
    S.rot[1] = -std::sin(yaw);
    S.rot[2] = std::sin(yaw);
    S.rot[3] = std::cos(yaw);
    S.has_xform = !(S.trans[0] == 0.0 && S.trans[1] == 0.0 && S.rot[0] == 1.0 && S.rot[1] == 0.0 && S.rot[2] == 0.0 &&
                    S.rot[3] == 1.0);
    S.radius = 1.0;
    S.rout = 1e300;
    S.prune_scale = 1.0;
    S.prune_rmin = 0.0;
    if (cfg.mesh_faces && cfg.mesh_nf > 0) {  // triangle-mesh functor requested: overrides the registry name
        S.id = SH_MESH;
        return;
    }
    {
        // Circumradius of each analytic shape about its own origin, rounded up with a 0.05 margin (measured: the largest
        // |q| with sdf(q) <= 0; the functors are exact distances outside the shape, so sdf(q) >= |q| - R everywhere —
        // tests/test_oracle_shapes.py::test_circumradius_bound checks every entry against the oracle, the GPU parity
        // tests check the pruned scan bit for bit).  The body-frame pre-transform shifts the origin by |trans|.
        static const double kRout[17] = {2.85, 2.36, 3.05, 3.05, 2.88, 2.97, 5.05, 3.65, 4.55, 4.63, 2.42, 3.84, 2.05, 4.52, 3.05, 6.05, 1.05};
        if (S.id >= 0 && S.id <= SH_CIRCLE) S.rout = kRout[S.id] + std::sqrt(S.trans[0] * S.trans[0] + S.trans[1] * S.trans[1]);
    }
    switch (S.id) {
        case SH_HORSESHOE: S.cst[0] = std::cos(20.5); S.cst[1] = std::sin(20.5); break;  // Shape.hpp:855
        case SH_PIE: S.cst[0] = std::cos(43.0); S.cst[1] = std::sin(43.0); break;        // :1235
        case SH_PIE2: S.cst[0] = std::cos(1.0); S.cst[1] = std::sin(1.0); break;         // :1276
        case SH_ARC: S.cst[0] = std::sin(20.0); S.cst[1] = std::cos(20.0); break;        // :1320
        case SH_CUTDISK: S.cst[0] = std::sqrt(5.0 * 5.0 - 2.0 * 2.0); break;             // :701
        case SH_HEART: S.cst[0] = std::sqrt(2.0) / 4.0; break;                           // :946
        case SH_VESICA: {                                                                // :1119-1128
            const double ax = 2, ay = 4, bx = -2, by = -4, w = 0.8;
            const double bax = bx - ax, bay = by - ay;
            const double r = 0.5 * std::sqrt(bax * bax + bay * bay);
            S.cst[0] = r;
            S.cst[1] = 0.5 * (r * r - w * w) / w;
            S.cst[2] = bax / r;
            S.cst[3] = bay / r;
            break;
        }
        case SH_MOON: {  // :1205-1206
            const double d = 0.8, ra = 3.0, rb = 2.4;
            const double a = (ra * ra - rb * rb + d * d) / (2.0 * d);
            S.cst[0] = a;
            S.cst[1] = std::sqrt(std::max(ra * ra - a * a, 0.0));
            break;
        }
        case SH_UNEVENCAPSULE: {  // :535-536
            const double b = (2.0 - 1.0) / 5.0;
            S.cst[0] = b;
            S.cst[1] = std::sqrt(1.0 - b * b);
            break;
        }
        case SH_POLYGON: {
            const double rect[8] = {6, -0.1, 6, 0.1, -6, 0.1, -6, -0.1};  // sw_manager.hpp:365-369
            const double *xy = rect;
            int n = 4;
            if (cfg.polygon_xy && cfg.polygon_n >= 3 && cfg.polygon_n <= kMaxPolyEdges) {
                xy = cfg.polygon_xy;
                n = cfg.polygon_n;
            }
            S.poly_n = n;
            for (int i = 0; i < n; ++i) {  // Polygon ctor, Shape.hpp:1429-1446
                const int j = (i + 1) % n;
                S.poly_sx[i] = xy[2 * i];
                S.poly_sy[i] = xy[2 * i + 1];
                S.poly_ex[i] = xy[2 * j];
                S.poly_ey[i] = xy[2 * j + 1];
            }
            S.has_xform = 0;
            S.rout = 0.0;  // Polygon ignores trans/Rotate: the farthest vertex bounds it
            for (int i = 0; i < n; ++i) S.rout = std::max(S.rout, std::sqrt(xy[2 * i] * xy[2 * i] + xy[2 * i + 1] * xy[2 * i + 1]));
            S.rout += 0.05;
            break;
        }
        default: break;
    }
}

// The test hooks of the environment (TestHooks), read once per context
TestHooks read_test_hooks() {
    TestHooks h;
    if (const char *fg = std::getenv("SVSDF_FORCE_GRID_OUTER")) h.force_grid_outer = std::atoi(fg);
    if (const char *fb = std::getenv("SVSDF_FORCE_BATCHED")) h.force_batched = std::atoi(fb);
    if (const char *fw = std::getenv("SVSDF_FORCE_GSIP_WIDE")) h.force_gsip_wide = std::atoi(fw);
    if (const char *fg = std::getenv("SVSDF_FORCE_GRID_GSIP")) h.force_grid_gsip = std::atoi(fg);
    if (const char *fg = std::getenv("SVSDF_FORCE_GRID_ASTAR")) h.force_grid_astar = std::atoi(fg);
    if (const char *fp = std::getenv("SVSDF_FORCE_POSE_WINDOWS")) h.force_pose_windows = std::atoi(fp);
    if (const char *fc = std::getenv("SVSDF_FORCE_OUTER_CHUNK")) h.force_outer_chunk = std::atoi(fc);
    return h;
}

// The mesh functor's device arrays (SH_MESH): the transformed face soup, the winding-number hierarchy and the far-field bound of
// choiceTInit's layer-1 pruning.  CUDA errors are reported on stderr like svsdf_create's own.
int upload_mesh(svsdf_ctx *ctx, const svsdf_config &cfg) {
    auto fail = [](cudaError_t e) {
        std::fprintf(stderr, "svsdf_create: %s\n", cudaGetErrorString(e));
        return SVSDF_ERR_CUDA;
    };
    cudaError_t e;
    // BasicShape ctor (Shape.hpp:285-309): every vertex becomes R v + trans, then the per-face soup
    const ShapeParams &S = ctx->shape;
    const double R[3][3] = {{S.rot[0], S.rot[1], 0.0}, {S.rot[2], S.rot[3], 0.0}, {0.0, 0.0, 1.0}};
    const double tr[3] = {S.trans[0], S.trans[1], 0.0};
    std::vector<double> tri((size_t)cfg.mesh_nf * kMeshStride);
    for (int f = 0; f < cfg.mesh_nf; ++f) {
        double *rec = &tri[(size_t)f * kMeshStride];
        for (int k = 0; k < 3; ++k) {
            const double *v = cfg.mesh_vertices + 3 * (size_t)cfg.mesh_faces[3 * f + k];
            for (int j = 0; j < 3; ++j)
                rec[3 * k + j] = ((v[0] * R[j][0] + v[1] * R[j][1]) + v[2] * R[j][2]) + tr[j];
        }
        // rmax: farthest point of the face from vertex a (one of the other two vertices), padded upwards
        const double ab = std::sqrt((rec[3] - rec[0]) * (rec[3] - rec[0]) + (rec[4] - rec[1]) * (rec[4] - rec[1]) + (rec[5] - rec[2]) * (rec[5] - rec[2]));
        const double ac = std::sqrt((rec[6] - rec[0]) * (rec[6] - rec[0]) + (rec[7] - rec[1]) * (rec[7] - rec[1]) + (rec[8] - rec[2]) * (rec[8] - rec[2]));
        rec[9] = std::max(ab, ac) * (1.0 + 1e-12) + 1e-300;
    }
    auto up = [](auto &buf, const auto &v) -> cudaError_t {
        const cudaError_t e2 = buf.reserve(v.size());
        return e2 != cudaSuccess ? e2 : cudaMemcpy(buf, v.data(), v.size() * sizeof(v[0]), cudaMemcpyHostToDevice);
    };
    if ((e = up(ctx->mesh.d_tri, tri)) != cudaSuccess) return fail(e);
    ctx->shape.mesh_tri = ctx->mesh.d_tri;
    ctx->shape.mesh_nf = cfg.mesh_nf;
    ctx->shape.has_xform = 0;
    // the winding-number hierarchy over the SAME transformed vertices (fast_winding_number.cpp:380-408 is handed V after
    // the ctor's transform, Shape.hpp:303-309), built on the host and uploaded as four flat arrays
    std::vector<double> Vt((size_t)cfg.mesh_nv * 3);
    for (int i = 0; i < cfg.mesh_nv; ++i) {
        const double *v = cfg.mesh_vertices + 3 * (size_t)i;
        for (int j = 0; j < 3; ++j) Vt[3 * (size_t)i + j] = ((v[0] * R[j][0] + v[1] * R[j][1]) + v[2] * R[j][2]) + tr[j];
    }
    host::FwnBvh B;
    B.build(Vt.data(), cfg.mesh_nv, cfg.mesh_faces, cfg.mesh_nf);
    if (B.nn < 1 || B.depth() > kFwnMaxDepth) {
        ctx->err = "svsdf_create: mesh hierarchy deeper than kFwnMaxDepth";
        return SVSDF_ERR_INVALID;
    }
    // child boxes for the closest-triangle descent: lo x, lo y, hi x, hi y two ulps outwards (the float boxes then contain
    // the double vertices), squared z gap to the query plane z = 0 rounded down, pad
    std::vector<float> cb(B.cbox.size(), 0.0f);
    float boxmag = 0.0f;
    {
        const float ninf = -std::numeric_limits<float>::infinity(), pinf = std::numeric_limits<float>::infinity();
        auto out = [&](float v, float dir) { return std::isfinite(v) ? std::nextafter(std::nextafter(v, dir), dir) : v; };
        for (size_t k = 0; k + 5 < cb.size(); k += 6) {
            const float *b = &B.cbox[k];  // min xyz, max xyz
            const float lox = out(b[0], ninf), loy = out(b[1], ninf), loz = out(b[2], ninf), hix = out(b[3], pinf), hiy = out(b[4], pinf),
                        hiz = out(b[5], pinf);
            cb[k] = lox; cb[k + 1] = loy; cb[k + 2] = hix; cb[k + 3] = hiy;
            const double gz = std::max(std::max((double)loz, -(double)hiz), 0.0);
            float dz2 = (float)(gz * gz);
            if ((double)dz2 > gz * gz) dz2 = std::nextafter(dz2, 0.0f);
            cb[k + 4] = std::isfinite(dz2) ? dz2 : 0.0f;
            for (int j = 0; j < 4; ++j)
                if (std::isfinite(cb[k + j])) boxmag = std::max(boxmag, std::fabs(cb[k + j]));
        }
    }
    ctx->shape.fwn_boxmag = boxmag;
    std::vector<float> tf((size_t)cfg.mesh_nf * 12, 0.0f);
    for (int f = 0; f < cfg.mesh_nf; ++f)
        for (int k = 0; k < 3; ++k)
            for (int j = 0; j < 3; ++j) tf[12 * (size_t)f + 3 * k + j] = B.U[3 * (size_t)B.F[3 * f + k] + j];
    if ((e = up(ctx->mesh.d_fwn_child, B.child)) != cudaSuccess) return fail(e);
    if ((e = up(ctx->mesh.d_fwn_data, B.data)) != cudaSuccess) return fail(e);
    if ((e = up(ctx->mesh.d_fwn_cbox, cb)) != cudaSuccess) return fail(e);
    if ((e = up(ctx->mesh.d_fwn_trif, tf)) != cudaSuccess) return fail(e);
    // Far-field bound for choiceTInit's layer-1 pruning (thread_choice_t_init): sdf = (1 - 2 w) d with d >= |q| - Rv (Rv: the
    // largest vertex norm; the query has z = 0, the origin is the body origin).  Beyond rho0 = max_i(|P_i| + 2 sqrt(maxPDist2_i))
    // none of the root's children is entered, w is the sum of their four expansions / (4 pi), and each expansion is bounded
    // term by term through the magnitudes of its coefficients (|q^| <= 1 componentwise) and |q - P_i| >= rho0 - |P_i|:
    //   |order 0| <= |N|_1 m^2,  |order 1| <= (|tr| + 3 (sum of |Nij| rows)) m^3,  |order 2| <= (1.5 A + 7.5 B) m^4,  m = 1 / (rho0 - |P_i|).
    // With omega that bound (padded 2 % for the float rounding of the evaluation), sdf >= (1 - 2 omega)(|q| - Rv) for |q| >= rho0.
    {
        double Rv = 0.0;
        for (int i = 0; i < cfg.mesh_nv; ++i)
            Rv = std::max(Rv, std::sqrt(Vt[3 * (size_t)i] * Vt[3 * (size_t)i] + Vt[3 * (size_t)i + 1] * Vt[3 * (size_t)i + 1] + Vt[3 * (size_t)i + 2] * Vt[3 * (size_t)i + 2]));
        double rho0 = 0.0;
        int nchild = 0;
        for (int i = 0; i < 4; ++i) {
            if (B.child[i] == host::FwnBvh::EMPTY) break;
            ++nchild;
            const double Pn = std::sqrt((double)B.row(0, 1)[i] * B.row(0, 1)[i] + (double)B.row(0, 2)[i] * B.row(0, 2)[i] + (double)B.row(0, 3)[i] * B.row(0, 3)[i]);
            rho0 = std::max(rho0, Pn + 2.0 * std::sqrt(std::max(0.0, (double)B.row(0, 0)[i])));
        }
        rho0 = std::max(rho0, Rv) * (1.0 + 1e-4) + 1e-6;
        double omega = 0.0;
        bool finite = std::isfinite(rho0);
        for (int i = 0; i < nchild && finite; ++i) {
            auto a = [&](int r) { return std::fabs((double)B.row(0, r)[i]); };
            const double Pn = std::sqrt((double)B.row(0, 1)[i] * B.row(0, 1)[i] + (double)B.row(0, 2)[i] * B.row(0, 2)[i] + (double)B.row(0, 3)[i] * B.row(0, 3)[i]);
            const double m = 1.0 / (rho0 - Pn);
            const double A0 = a(4) + a(5) + a(6);
            const double A1 = std::fabs((double)B.row(0, 7)[i] + B.row(0, 8)[i] + B.row(0, 9)[i]) + 3.0 * (a(7) + a(8) + a(9) + a(10) + a(11) + a(12));
            const double t0 = std::fabs((double)B.row(0, 20)[i] + B.row(0, 21)[i]) + std::fabs((double)B.row(0, 22)[i] + B.row(0, 17)[i]) +
                              std::fabs((double)B.row(0, 18)[i] + B.row(0, 19)[i]);
            const double t1 = a(17) + a(18) + a(19) + a(20) + a(21) + a(22);
            const double A2 = 1.5 * (3.0 * (a(13) + a(14) + a(15)) + t0) + 7.5 * (a(13) + a(14) + a(15) + a(16) + t1);
            omega += A0 * m * m + A1 * m * m * m + A2 * m * m * m * m;
            finite = finite && std::isfinite(omega);
        }
        omega = omega / (4.0 * 3.14159265358979323846) * 1.02 + 1e-6;
        if (finite && omega < 0.45) {
            ctx->shape.rout = Rv * (1.0 + 1e-9) + 1e-9;
            ctx->shape.prune_scale = 1.0 / (1.0 - 2.0 * omega);
            ctx->shape.prune_rmin = rho0;
        }
    }
    ctx->shape.fwn_nn = B.nn;
    ctx->shape.fwn_child = ctx->mesh.d_fwn_child;
    ctx->shape.fwn_data = ctx->mesh.d_fwn_data;
    ctx->shape.fwn_cbox = ctx->mesh.d_fwn_cbox;
    ctx->shape.fwn_trif = ctx->mesh.d_fwn_trif;
    return SVSDF_OK;
}

}  // namespace

bool scale_valid(const svsdf_scale &z) {
    for (int d = 0; d < 2; ++d) {
        const double v[4] = {z.a[d], z.b[d], z.w[d], z.phi[d]};
        for (double x : v)
            if (!std::isfinite(x)) return false;
        // s_d(t) stays in [kScaleMin, kScaleMax] at every t (|sin| <= 1, rounding is monotone), so fl(sy * sx) is a normal
        // number and the cofactor inverse 1/fl(sy * sx) and St^-1 are finite and non-zero.  a_d - |b_d| > 0 alone is not
        // enough: a = 1e-160 makes fl(sy * sx) subnormal and 1/det = inf, a = 1e160 makes it inf and St^-1 = 0
        if (!(z.a[d] - std::fabs(z.b[d]) >= kScaleMin && z.a[d] + std::fabs(z.b[d]) <= kScaleMax)) return false;
        if (!(std::fabs(z.w[d]) * kMaxDuration + std::fabs(z.phi[d]) < 1e6)) return false;
    }
    return true;
}

bool dynamics_valid(const svsdf_dynamics &d) {
    const double v[5] = {d.vmax, d.omgmax, d.weight_v, d.weight_omg, d.smoothingEps};
    for (double e : v)
        if (!std::isfinite(e)) return false;
    return d.vmax > 0.0 && d.omgmax > 0.0 && d.weight_v >= 0.0 && d.weight_omg >= 0.0 && d.smoothingEps > 0.0 && d.integralIntervs >= 1 &&
           d.integralIntervs <= 64;
}
host::DynamicsParams to_host_dynamics(const svsdf_dynamics &d) {
    host::DynamicsParams p;
    p.vmax = d.vmax; p.omgmax = d.omgmax; p.weight_v = d.weight_v; p.weight_omg = d.weight_omg; p.eps = d.smoothingEps;
    p.res = d.integralIntervs;
    return p;
}

static bool pose_penalty_valid(const svsdf_pose_penalty &p) {
    const double v[4] = {p.weight, p.half[0], p.half[1], p.half[2]};
    for (double e : v)
        if (!std::isfinite(e)) return false;
    return p.weight >= 0.0 && p.integralIntervs >= 1 && p.integralIntervs <= 64 && p.half[0] > 0.0 && p.half[1] > 0.0 && p.half[2] > 0.0;
}

int pose_penalty_check(svsdf_ctx *ctx, const svsdf_pose_penalty &p, const char *who) {
    if (!pose_penalty_valid(p)) {
        ctx->err = std::string(who) + ": needs finite values, weight >= 0, 1 <= integralIntervs <= 64 and half sizes > 0";
        return SVSDF_ERR_INVALID;
    }
    if (ctx->shape.id == SH_MESH) {
        ctx->err = std::string(who) + ": not available for the mesh functor";
        return SVSDF_ERR_INVALID;
    }
    return SVSDF_OK;
}

extern "C" {

void svsdf_default_config(svsdf_config *cfg) {
    std::memset(cfg, 0, sizeof(*cfg));
    cfg->shape = "star";
    cfg->weight_p = 60.0;
    cfg->safety_hor = 0.7;
    cfg->rho = 3.8;
    cfg->strict_fp = 1;  // reference-rounding build is the default
}

int svsdf_shape_id(const char *name) { return shape_id_from_name(name); }
int svsdf_shape_bound_radius(const svsdf_config *cfg, double *radius_out) {
    if (!cfg || !radius_out) return SVSDF_ERR_INVALID;
    ShapeParams S;
    build_shape(*cfg, S);
    *radius_out = S.rout;
    return SVSDF_OK;
}

int svsdf_create(const svsdf_config *cfg, svsdf_ctx **out) {
    if (!cfg || !out) return SVSDF_ERR_INVALID;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return SVSDF_ERR_CUDA;  // no CPU fallback
    if (cfg->device < 0 || cfg->device >= ndev) return SVSDF_ERR_INVALID;
    if (cfg->polygon_xy && (cfg->polygon_n < 3 || cfg->polygon_n > kMaxPolyEdges)) return SVSDF_ERR_INVALID;
    if (cfg->mesh_nf < 0 || cfg->mesh_nv < 0 || cfg->mesh_nf > kMaxMeshFaces) return SVSDF_ERR_INVALID;
    if (cfg->mesh_nf > 0) {
        if (!cfg->mesh_faces || !cfg->mesh_vertices || cfg->mesh_nv < 3) return SVSDF_ERR_INVALID;
        for (int64_t k = 0; k < 3 * (int64_t)cfg->mesh_nf; ++k)
            if (cfg->mesh_faces[k] < 0 || cfg->mesh_faces[k] >= cfg->mesh_nv) return SVSDF_ERR_INVALID;
    }
    svsdf_ctx *ctx = new svsdf_ctx();
    ctx->cfg = *cfg;
    ctx->shape_name = cfg->shape ? cfg->shape : "";
    ctx->cfg.shape = ctx->shape_name.c_str();
    build_shape(*cfg, ctx->shape);
    ctx->cp.weight_p = cfg->weight_p;
    ctx->cp.safety_hor = cfg->safety_hor;
    ctx->rho = cfg->rho;
    ctx->device = cfg->device;
    ctx->strict = cfg->strict_fp != 0;
    ctx->hooks = read_test_hooks();
    auto fail = [&](cudaError_t e) {
        std::fprintf(stderr, "svsdf_create: %s\n", cudaGetErrorString(e));
        svsdf_destroy(ctx);
        return SVSDF_ERR_CUDA;
    };
    cudaError_t e;
    if ((e = cudaSetDevice(ctx->device)) != cudaSuccess) return fail(e);
    cudaDeviceProp prop;
    if ((e = cudaGetDeviceProperties(&prop, ctx->device)) != cudaSuccess) return fail(e);
    if (prop.major != 9 || prop.minor != 0) {  // sm_90a code loads on compute capability 9.0 only
        std::fprintf(stderr, "svsdf_create: device sm_%d%d is not a Hopper H100 (kernels are built for sm_90a only)\n",
                     prop.major, prop.minor);
        svsdf_destroy(ctx);
        return SVSDF_ERR_CUDA;
    }
    ctx->sm_count = prop.multiProcessorCount;
    if ((e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess) return fail(e);
    if ((e = cudaEventCreate(&ctx->ev0)) != cudaSuccess) return fail(e);
    if ((e = cudaEventCreate(&ctx->ev1)) != cudaSuccess) return fail(e);
    for (int k = 0; k < 5; ++k)
        if ((e = cudaEventCreate(&ctx->evk[k])) != cudaSuccess) return fail(e);
    if ((e = ctx->d_n_inside.reserve(1)) != cudaSuccess) return fail(e);
    if ((e = ctx->d_eval_counter.reserve(1)) != cudaSuccess) return fail(e);
    if ((e = ctx->d_ticket.reserve(1)) != cudaSuccess) return fail(e);
    cudaMemset(ctx->d_ticket, 0, sizeof(unsigned int));
    cudaMemset(ctx->d_n_inside, 0, sizeof(int));
    cudaMemset(ctx->d_eval_counter, 0, sizeof(unsigned long long));
    ctx->cfg.mesh_vertices = nullptr;  // caller's arrays are not kept
    ctx->cfg.mesh_faces = nullptr;
    ctx->cfg.polygon_xy = nullptr;
    if (ctx->shape.id == SH_MESH) {
        if (const int rc = upload_mesh(ctx, *cfg)) {
            svsdf_destroy(ctx);
            return rc;
        }
    }
    *out = ctx;
    return SVSDF_OK;
}

void svsdf_destroy(svsdf_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    if (ctx->lmbm) svsdf_lmbm_close(ctx->lmbm);
    if (ctx->upload.ev) cudaEventDestroy(ctx->upload.ev);
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    for (int k = 0; k < 5; ++k)
        if (ctx->evk[k]) cudaEventDestroy(ctx->evk[k]);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;  // the buffers free themselves
}

const char *svsdf_last_error(const svsdf_ctx *ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int svsdf_set_points(svsdf_ctx *ctx, const double *pts, int64_t P, int stride) {
    if (!ctx || P < 0 || stride < 2 || (P > 0 && !pts)) return SVSDF_ERR_INVALID;
    if (P > 2000000000LL) { ctx->err = "svsdf: too many points"; return SVSDF_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    ctx->points_ext = nullptr;
    CK(ctx->points_buf.reserve((size_t)P * 2));  // never null, also for P == 0
    if (ctx->upload.inflight) {  // the previous upload still reads the stage
        CK(cudaEventSynchronize(ctx->upload.ev));
        ctx->upload.inflight = false;
    }
    if (!ctx->upload.ev) CK(cudaEventCreateWithFlags(&ctx->upload.ev, cudaEventDisableTiming));
    CK(ctx->upload.h_stage.reserve((size_t)P * 2));
    double *h = ctx->upload.h_stage;
    // pos_eva(2) = 0 (back_end_optimizer.hpp:791): only x, y are kept.  Packed into the pinned stage chunk by chunk by a few
    // host threads; every chunk is handed to the copy engine as soon as it is packed (packing of the next chunks overlaps the
    // DMA of the finished ones).  One thread for small inputs.
    const int64_t chunk = 16384;
    const int64_t nchunks = (P + chunk - 1) / chunk;
    int nth = (int)std::min<int64_t>(nchunks, 4);
#ifdef _OPENMP
    nth = std::max(1, std::min(nth, omp_get_num_procs()));  // not omp_get_max_threads(): launchers set OMP_NUM_THREADS = 1 per rank
#else
    nth = 1;
#endif
    int first_err = (int)cudaSuccess;
    const int dev = ctx->device;
    double *d_points = ctx->points_buf;
    cudaStream_t stream = ctx->stream;
#pragma omp parallel num_threads(nth) if (nth > 1)
    {
        if (nth > 1) cudaSetDevice(dev);  // the worker threads' current device
#pragma omp for schedule(dynamic, 1)
        for (int64_t c = 0; c < nchunks; ++c) {
            const int64_t b = c * chunk, e = std::min(P, b + chunk);
            pack_xy(h + 2 * b, pts + b * stride, e - b, stride);
            cudaError_t ce = cudaMemcpyAsync(d_points + 2 * b, h + 2 * b, (size_t)(e - b) * 2 * sizeof(double), cudaMemcpyHostToDevice, stream);
            if (ce != cudaSuccess) {
#pragma omp atomic write
                first_err = (int)ce;
            }
        }
    }
    if (first_err != (int)cudaSuccess) {
        ctx->err = std::string("svsdf_set_points: cudaMemcpyAsync: ") + cudaGetErrorString((cudaError_t)first_err);
        return SVSDF_ERR_CUDA;
    }
    CK(cudaEventRecord(ctx->upload.ev, ctx->stream));  // no wait here: see svsdf_ctx::upload
    ctx->upload.inflight = true;
    ctx->P = P;
    ctx->last_n_inside = -1;
    return ensure_scratch(ctx, P);
}

int svsdf_set_points_device(svsdf_ctx *ctx, const double *dev_xy, int64_t P) {
    if (!ctx || P < 0 || (P > 0 && !dev_xy)) return SVSDF_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    ctx->points_buf.release();
    ctx->points_ext = dev_xy;
    ctx->P = P;
    return ensure_scratch(ctx, P);
}

int svsdf_device_ptr_points(svsdf_ctx *ctx, const double **dev_xy) {
    if (!ctx || !dev_xy) return SVSDF_ERR_INVALID;
    if (ctx->upload.inflight) {  // the pointer may be used on other streams: the upload has to be complete
        CK(cudaSetDevice(ctx->device));
        CK(cudaEventSynchronize(ctx->upload.ev));
        ctx->upload.inflight = false;
    }
    *dev_xy = ctx->points();
    return SVSDF_OK;
}

int svsdf_get_points(svsdf_ctx *ctx, double *xy_out, int64_t capacity, int64_t *n_points) {
    if (!ctx) return SVSDF_ERR_INVALID;
    if (n_points) *n_points = ctx->P;
    if (!xy_out || capacity <= 0 || ctx->P == 0) return SVSDF_OK;
    CK(cudaSetDevice(ctx->device));
    const int64_t n = ctx->P < capacity ? ctx->P : capacity;
    CK(cudaMemcpy(xy_out, ctx->points(), (size_t)n * 2 * sizeof(double), cudaMemcpyDeviceToHost));
    return SVSDF_OK;
}

int svsdf_set_scale(svsdf_ctx *ctx, const svsdf_scale *scale) {
    if (!ctx) return SVSDF_ERR_INVALID;
    if (!scale) {
        ctx->scaled = false;
        return SVSDF_OK;
    }
    if (!scale_valid(*scale)) {
        ctx->err = "svsdf_set_scale: schedule must be finite with a_d - |b_d| >= 1e-6, a_d + |b_d| <= 1e6 and |w_d| * 300 + |phi_d| < 1e6";
        return SVSDF_ERR_INVALID;
    }
    for (int d = 0; d < 2; ++d) {
        ctx->sched.a[d] = scale->a[d];
        ctx->sched.b[d] = scale->b[d];
        ctx->sched.w[d] = scale->w[d];
        ctx->sched.phi[d] = scale->phi[d];
    }
    ctx->scaled = true;
    return SVSDF_OK;
}

int svsdf_set_dynamics(svsdf_ctx *ctx, const svsdf_dynamics *dyn) {
    if (!ctx) return SVSDF_ERR_INVALID;
    if (!dyn) {
        ctx->dyn_on = false;
        return SVSDF_OK;
    }
    if (!dynamics_valid(*dyn)) {
        ctx->err = "svsdf_set_dynamics: needs finite values, vmax > 0, omgmax > 0, weights >= 0, smoothingEps > 0 and 1 <= integralIntervs <= 64";
        return SVSDF_ERR_INVALID;
    }
    ctx->dyn = to_host_dynamics(*dyn);
    ctx->dyn_on = true;
    return SVSDF_OK;
}

int svsdf_set_pose_penalty(svsdf_ctx *ctx, const svsdf_pose_penalty *p) {
    if (!ctx) return SVSDF_ERR_INVALID;
    if (!p) {
        ctx->pose_on = false;
        return SVSDF_OK;
    }
    if (const int rc = pose_penalty_check(ctx, *p, "svsdf_set_pose_penalty")) return rc;
    ctx->pose.weight = p->weight;
    ctx->pose.res = p->integralIntervs;
    for (int a = 0; a < 3; ++a) ctx->pose_half[a] = p->half[a];
    ctx->pose_on = true;
    return SVSDF_OK;
}

static int shape_eval(svsdf_ctx *ctx, int64_t n, const double *rel, double *out, int grad) {
    if (!ctx || n < 0 || (n > 0 && (!rel || !out))) return SVSDF_ERR_INVALID;
    if (n == 0) return SVSDF_OK;
    CK(cudaSetDevice(ctx->device));
    const int ow = grad ? 3 : 1;
    CK(ctx->h_stage.reserve((size_t)n * (2 + ow) * sizeof(double)));
    DeviceBuffer<double> d_in, d_out;
    CK(d_in.reserve((size_t)n * 2));
    CK(d_out.reserve((size_t)n * ow));
    double *h = reinterpret_cast<double *>(ctx->h_stage.get());
    pack_xy(h, rel, n, 3);
    CK(cudaMemcpyAsync(d_in, h, (size_t)n * 2 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    CK(kernels(ctx).shape_eval(ctx->shape, d_in, n, d_out, grad, ctx->stream));
    ctx->launches += 1;
    double *ho = h + 2 * n;
    CK(cudaMemcpyAsync(ho, d_out, (size_t)n * ow * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    std::memcpy(out, ho, (size_t)n * ow * sizeof(double));
    return SVSDF_OK;
}
int svsdf_shape_sdf(svsdf_ctx *ctx, int64_t n, const double *rel, double *sdf_out) { return shape_eval(ctx, n, rel, sdf_out, 0); }
int svsdf_shape_grad1(svsdf_ctx *ctx, int64_t n, const double *rel, double *grad3_out) { return shape_eval(ctx, n, rel, grad3_out, 1); }

int svsdf_sincos(svsdf_ctx *ctx, int64_t n, const double *x, double *sin_out, double *cos_out) {
    if (!ctx || n < 0 || (n > 0 && (!x || !sin_out || !cos_out))) return SVSDF_ERR_INVALID;
    if (n == 0) return SVSDF_OK;
    CK(cudaSetDevice(ctx->device));
    DeviceBuffer<double> d;
    CK(d.reserve((size_t)n * 3));
    CK(cudaMemcpyAsync(d, x, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    CK(kernels(ctx).sincos(d, n, d + n, d + 2 * n, ctx->stream));
    ctx->launches += 1;
    CK(cudaMemcpyAsync(sin_out, d + n, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(cos_out, d + 2 * n, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return SVSDF_OK;
}

int svsdf_last_kernel_ms(const svsdf_ctx *ctx, float *out4) {
    if (!ctx || !out4) return SVSDF_ERR_INVALID;
    for (int k = 0; k < 4; ++k) out4[k] = ctx->last_kernel_ms[k];
    return SVSDF_OK;
}

int svsdf_kernel_launches(const svsdf_ctx *ctx, int64_t *count) {
    if (!ctx || !count) return SVSDF_ERR_INVALID;
    *count = ctx->launches;
    return SVSDF_OK;
}

int svsdf_executed_evals(svsdf_ctx *ctx, int enable, uint64_t *count) {
    if (!ctx) return SVSDF_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    if (count) {
        unsigned long long v = 0;
        CK(cudaStreamSynchronize(ctx->stream));
        CK(cudaMemcpy(&v, ctx->d_eval_counter, sizeof(v), cudaMemcpyDeviceToHost));
        *count = v;
    }
    ctx->count_evals = enable != 0;
    CK(cudaMemset(ctx->d_eval_counter, 0, sizeof(unsigned long long)));
    return SVSDF_OK;
}

int svsdf_fp64_peak(svsdf_ctx *ctx, double *tflops) {
    if (!ctx || !tflops) return SVSDF_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    const int grid = ctx->sm_count * 8, iters = 1 << 16;
    DeviceBuffer<double> d;
    CK(d.reserve((size_t)grid * 256));
    float best = 1e30f;
    for (int r = 0; r < 5; ++r) {
        CK(cudaEventRecord(ctx->ev0, ctx->stream));
        CK(fast::launch_fp64_peak(d, grid, iters, ctx->stream));
        CK(cudaEventRecord(ctx->ev1, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
        if (r > 0 && ms < best) best = ms;
        ctx->launches += 1;
    }
    const double flops = 2.0 * 8.0 * (double)iters * (double)grid * 256.0;
    *tflops = flops / (best * 1e-3) / 1e12;
    return SVSDF_OK;
}

}  // extern "C"
