// svsdf_runtime_swept.cpp — the swept volume's outline (svsdf_swept_contour) and the map clearance of one or n trajectories
// (svsdf_map_clearance[_multi]), which share the path samples of the band bound.  Kernels: svsdf_swept.cu, svsdf_clearance.cu.
#include <algorithm>
#include <cmath>
#include <cstdlib>

#include "svsdf_runtime.h"

extern "C" {

// ---- svsdf_swept_contour (kernels: svsdf_swept.cu; the band bound: DESIGN.md §7) ----------------------------------------------
namespace {
constexpr int64_t kSweptDefaultCorners = (int64_t)1 << 25;
constexpr int64_t kSweptMaxCorners = (int64_t)1 << 28;  // vertex, segment and triangle indices stay in int32

// Path samples for the band bound.  Piece i is cut into ceil(T_i / 0.15) equal parts of local time; a sample is the position at a
// part's midpoint (the piece's own polynomial) and delta = half the part (plus a rounding allowance on the local time) times a bound
// on |velocity| over the piece from the coefficients: |v_d| <= sum_k k |c_dk| Tmax^(k-1).  reach = (delta + s_eff rho) padded, where a
// body-frame point beyond rho is provably > iso.  Sampling piece by piece needs no continuity between pieces.
void swept_samples(const svsdf_ctx *ctx, int N, const double *T, const double *coeffs, double D, double rho, std::vector<double> &samp) {
    double s_eff = 1.0;
    if (ctx->scaled)
        for (int d = 0; d < 2; ++d) s_eff = std::max(s_eff, ctx->sched.a[d] + std::fabs(ctx->sched.b[d]));
    const double ext = 1e-9 * (1.0 + D);
    samp.clear();
    for (int i = 0; i < N; ++i) {
        const double *cx = coeffs + 6 * i, *cy = coeffs + 6 * N + 6 * i;
        const double tmax = T[i] * (1.0 + 1e-9) + ext;
        double vx = 0.0, vy = 0.0, tk = 1.0;
        for (int k = 1; k < 6; ++k) {
            vx += k * std::fabs(cx[k]) * tk;
            vy += k * std::fabs(cy[k]) * tk;
            tk *= tmax;
        }
        const double vmax = std::sqrt(vx * vx + vy * vy);
        const int m = std::max(1, (int)std::ceil(T[i] / 0.15));
        const double part = T[i] / m;
        for (int j = 0; j < m; ++j) {
            const double tau = (j + 0.5) * part;
            double x = 0.0, y = 0.0, tn = 1.0;
            for (int k = 0; k < 6; ++k) {
                x += cx[k] * tn;
                y += cy[k] * tn;
                tn *= tau;
            }
            const double delta = (0.5 * part + ext) * vmax;
            const double reach = (delta + s_eff * rho) * (1.0 + 1e-9) + 1e-9 * (1.0 + std::fabs(x) + std::fabs(y) + s_eff * rho);
            samp.push_back(x);
            samp.push_back(y);
            samp.push_back(reach);
        }
    }
}

// largest i with fl(i h) <= x / smallest i with fl(i h) >= x
int64_t lattice_floor(double x, double h) {
    int64_t i = (int64_t)std::floor(x / h);
    while ((double)i * h > x) --i;
    while ((double)(i + 1) * h <= x) ++i;
    return i;
}
int64_t lattice_ceil(double x, double h) {
    int64_t i = (int64_t)std::ceil(x / h);
    while ((double)i * h < x) ++i;
    while ((double)(i - 1) * h >= x) --i;
    return i;
}

// svsdf_swept_contour (multi = false, n = 1, status_out unused: the status is returned) and svsdf_swept_contour_multi: every check
// before any launch, then the mesher's kernels over the concatenation of the n problems (svsdf_swept.cu) in one set of launches.  The
// outer solve of the needed corners is the single call's own (run_kernels, outer only) or, for n problems, the multi-problem one
// (run_multi, outer only), which gives every point the same bits.
int swept_run(svsdf_ctx *ctx, bool multi, int n, const svsdf_clearance_problem *problems, const svsdf_swept_params *prm,
              svsdf_swept_mesh *out, int *status_out) {
    const std::string who = multi ? "svsdf_swept_contour_multi" : "svsdf_swept_contour";
    auto invalid = [&](const std::string &msg) {
        ctx->err = msg;
        return SVSDF_ERR_INVALID;
    };
    const double h = prm->h, iso = prm->iso;
    if (!(std::isfinite(h) && h > 0.0)) return invalid(who + ": h must be finite and > 0");
    if (!std::isfinite(iso)) return invalid(who + ": iso must be finite");
    const int64_t cap = prm->max_corners == 0 ? kSweptDefaultCorners : prm->max_corners;
    if (cap < 4 || cap > kSweptMaxCorners) return invalid(who + ": max_corners must be 0 or in 4 .. 2^28");
    if (prm->has_box) {
        const double *b = prm->box;
        if (!(std::isfinite(b[0]) && std::isfinite(b[1]) && std::isfinite(b[2]) && std::isfinite(b[3]))) return invalid(who + ": non-finite box");
        if (b[0] > b[2] || b[1] > b[3]) return invalid(who + ": inverted box");
    }
    // rho: body-frame radius beyond which the shape functor is provably > iso (sdf >= (|q| - R) / prune_scale for |q| >= prune_rmin)
    const ShapeParams &S = ctx->shape;
    const bool bounded = S.rout < 1e299;
    if (!prm->has_box && !bounded) return invalid(who + ": the shape has no far-field bound; give a box");
    const double rho = bounded ? std::max(std::max(S.prune_rmin, S.rout + S.prune_scale * iso), 0.0) : INFINITY;
    // per problem: its samples and grid; tiles and whole marching-squares blocks in problem order
    std::vector<SweptProblem> tab(n);
    std::vector<double> samp_all, samp;
    int64_t corners = 0, tiles = 0, blocks = 0;
    for (int k = 0; k < n; ++k) {
        const svsdf_clearance_problem &q = problems[k];
        const std::string at = multi ? who + ": problem " + std::to_string(k) + ": " : std::string();
        auto bad = [&](const std::string &msg) { return invalid(at + (multi ? msg : who + ": " + msg)); };
        BlobLayout L;
        double D = 0.0;
        const char *msg = nullptr;
        if (traj_layout(q.N, q.T, q.coeffs, L, D, &msg) != SVSDF_OK) return invalid(at + msg);
        for (int64_t e = 0; e < 18 * (int64_t)q.N; ++e)
            if (!std::isfinite(q.coeffs[e])) return bad("non-finite trajectory coefficient");
        swept_samples(ctx, q.N, q.T, q.coeffs, D, rho, samp);
        const int n_samp = (int)(samp.size() / 3);
        if (n_samp > kSweptMaxSamples) return bad("too many path samples");
        double bx0, by0, bx1, by1;
        if (prm->has_box) {
            bx0 = prm->box[0]; by0 = prm->box[1]; bx1 = prm->box[2]; by1 = prm->box[3];
        } else {
            bx0 = by0 = INFINITY;
            bx1 = by1 = -INFINITY;
            for (int s = 0; s < n_samp; ++s) {
                const double x = samp[3 * s], y = samp[3 * s + 1], r = samp[3 * s + 2];
                bx0 = std::min(bx0, x - r); bx1 = std::max(bx1, x + r);
                by0 = std::min(by0, y - r); by1 = std::max(by1, y + r);
            }
            // strictly beyond every reach, whatever the rounding of the subtractions above
            const double pad = 1e-9 * (1.0 + std::max(std::max(std::fabs(bx0), std::fabs(bx1)), std::max(std::fabs(by0), std::fabs(by1))));
            bx0 -= pad; by0 -= pad; bx1 += pad; by1 += pad;
        }
        const double lim = 0x1p50;
        if (!(std::fabs(bx0) / h < lim && std::fabs(bx1) / h < lim && std::fabs(by0) / h < lim && std::fabs(by1) / h < lim))
            return bad("box too large for the lattice of h");
        const int64_t i0 = lattice_floor(bx0, h), j0 = lattice_floor(by0, h);
        const int64_t i1 = std::max(lattice_ceil(bx1, h), i0 + 1), j1 = std::max(lattice_ceil(by1, h), j0 + 1);
        const int64_t nx64 = i1 - i0 + 1, ny64 = j1 - j0 + 1;
        if (nx64 > cap || ny64 > cap || nx64 * ny64 > cap) return bad("box has more corners than max_corners");
        SweptProblem &g = tab[k];
        std::memset(&g, 0, sizeof(g));
        g.i0 = i0; g.j0 = j0; g.nx = (int)nx64; g.ny = (int)ny64;
        g.tiles_x = (g.nx + kSweptTile - 1) / kSweptTile;
        g.nblk = (int)((nx64 * ny64 + kSweptBlock - 1) / kSweptBlock);
        g.tile0 = tiles;
        g.blk0 = blocks;
        g.samp0 = (int)(samp_all.size() / 3);
        g.n_samp = n_samp;
        samp_all.insert(samp_all.end(), samp.begin(), samp.end());
        tiles += (int64_t)g.tiles_x * ((g.ny + kSweptTile - 1) / kSweptTile);
        blocks += g.nblk;
        corners += nx64 * ny64;
    }
    // Band positions, the per-CTA prefixes (k_sw_scan) and the CTA indices are int32; tiles and blocks are no more than the corners.  A
    // single call (at most 2^28 corners) is never refused here.
    if (corners > 2147483647LL) return invalid(who + ": the problems' grids hold more than 2^31 - 1 corners");
    if (n == 0) return SVSDF_OK;
    CK(cudaSetDevice(ctx->device));

    SweptArgs A;
    std::memset(&A, 0, sizeof(A));
    A.n_prob = n;
    A.h = h; A.iso = iso;
    A.tiles = (int)tiles;
    A.n_blocks = (int)blocks;
    // per corner of the concatenation (whole blocks): need (1 byte), field (8), vertex ids (12)
    const size_t C = (size_t)blocks * kSweptBlock;
    const size_t off_field = align16(C), off_vid = off_field + align16(C * 8);
    CK(ctx->swept.d_corner.reserve(off_vid + C * 12));
    A.need = ctx->swept.d_corner;
    A.field = reinterpret_cast<double *>(ctx->swept.d_corner + off_field);
    A.vid = reinterpret_cast<int *>(ctx->swept.d_corner + off_vid);
    // small: header ([2..6] channel totals, [7] needed corners) | per-problem status [n][8] | problem table | samples (these four go up
    // in one copy) | tile counts | per-CTA counts
    const size_t off_stat = 64, off_tab = align16(off_stat + (size_t)n * 32), off_samp = align16(off_tab + tab.size() * sizeof(SweptProblem)),
                 up = off_samp + samp_all.size() * 8, off_tile = align16(up), off_blk = off_tile + align16((size_t)(tiles + 1) * 4);
    CK(ctx->swept.d_small.reserve(off_blk + (size_t)5 * (blocks + 1) * 4));
    int *d_hdr = reinterpret_cast<int *>(ctx->swept.d_small.get());
    A.stat = reinterpret_cast<int *>(ctx->swept.d_small + off_stat);
    A.prob = reinterpret_cast<const SweptProblem *>(ctx->swept.d_small + off_tab);
    A.samp = reinterpret_cast<double *>(ctx->swept.d_small + off_samp);
    A.tile_off = reinterpret_cast<int *>(ctx->swept.d_small + off_tile);
    A.blk = reinterpret_cast<int *>(ctx->swept.d_small + off_blk);
    CK(ctx->h_stage.reserve(up));
    std::memset(ctx->h_stage, 0, off_tab);
    std::memcpy(ctx->h_stage + off_tab, tab.data(), tab.size() * sizeof(SweptProblem));
    if (!samp_all.empty()) std::memcpy(ctx->h_stage + off_samp, samp_all.data(), samp_all.size() * 8);
    cudaStream_t st = ctx->stream;
    CK(cudaMemcpyAsync(ctx->swept.d_small, ctx->h_stage, up, cudaMemcpyHostToDevice, st));
    // classify the tiles and their corners, count and compact the needed corners
    CK(launch_swept(0, A, st));
    CK(launch_swept_scan(A.tile_off, A.tiles, 1, d_hdr + 7, st));
    std::vector<int> stat(8 * (size_t)n + 16);  // header, then the problems' status
    auto download_status = [&]() -> int {
        CK(cudaMemcpyAsync(ctx->h_stage, d_hdr, off_stat + (size_t)n * 32, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        std::memcpy(stat.data(), ctx->h_stage, off_stat + (size_t)n * 32);
        return SVSDF_OK;
    };
    int rc = download_status();
    if (rc) return rc;
    const int *pst = stat.data() + 16;  // problem k's status at pst[8 k]
    ctx->launches += 2;
    const int64_t P = stat[7];
    const size_t P1 = (size_t)std::max<int64_t>(P, 1);
    CK(ctx->swept.d_point.reserve(P1 * 32 + 32));
    A.P = P;
    A.pts = reinterpret_cast<double *>(ctx->swept.d_point.get());
    A.val = reinterpret_cast<double *>(ctx->swept.d_point + P1 * 16);
    A.idx = reinterpret_cast<int64_t *>(ctx->swept.d_point + P1 * 24);
    if (P > 0) {
        CK(launch_swept(1, A, st));
        double *val = const_cast<double *>(A.val);
        if (!multi) {
            // the outer solve of svsdf_query (outer_only = 1) on the mesher's own points: the same kernels, so the same bits per point
            rc = upload_traj(ctx, problems[0].N, problems[0].T, problems[0].coeffs, P);
            if (rc) return rc;
            rc = run_kernels(ctx, A.pts, P, false, false, val, nullptr, nullptr, nullptr);
            if (rc) return rc;
        } else {
            // the problems with needed corners, in problem order: their points are the concatenation's, in the same order; each keeps
            // the decomposition of its single call, and the outer solve's per-point values do not depend on it
            std::vector<MultiItem> items;
            for (int k = 0; k < n; ++k) {
                if (pst[8 * k + 7] == 0) continue;
                MultiItem it;
                it.N = problems[k].N; it.T = problems[k].T; it.coeffs = problems[k].coeffs; it.P = pst[8 * k + 7];
                items.push_back(it);
            }
            PointQuery pq{A.pts, val, nullptr};
            pq.outer_only = true;
            rc = run_multi(ctx, items.data(), (int)items.size(), nullptr, &pq);
            if (rc) return rc;
            for (const MultiItem &it : items)
                if (it.rc != SVSDF_OK) return invalid(who + ": a problem was refused by the evaluation");
        }
        CK(launch_swept(2, A, st));
        ctx->launches += 2;
    }
    // marching squares: counts, their prefix, then vertices, segments and triangles
    CK(launch_swept(3, A, st));
    CK(launch_swept_scan(A.blk, A.n_blocks, 5, d_hdr + 2, st));
    rc = download_status();
    if (rc) return rc;
    ctx->launches += 2;
    if (!multi && pst[0]) {
        ctx->err = "svsdf_swept_contour: non-finite field value";
        return SVSDF_ERR_NONFINITE;
    }
    // the outputs of every problem (the scan's int32 prefixes included) must stay in int32: one problem's always do (at most 2^28 corners)
    int64_t tot[5] = {0, 0, 0, 0, 0};
    for (int k = 0; k < n; ++k)
        for (int ch = 0; ch < 5; ++ch) tot[ch] += pst[8 * k + 2 + ch];
    for (int ch = 0; ch < 5; ++ch)
        if (tot[ch] > 2147483647LL) return invalid(who + ": the problems' outlines have more than 2^31 - 1 vertices, segments or triangles");
    const int64_t V = tot[0] + tot[1] + tot[2], Sg = tot[3], F = tot[4];
    const size_t b_verts = (size_t)V * 16, b_segs = (size_t)Sg * 8, b_tris = (size_t)F * 12;
    const size_t o_segs = align16(b_verts), o_tris = o_segs + align16(b_segs), o_end = o_tris + align16(b_tris);
    CK(ctx->swept.d_out.reserve(o_end + 16));
    A.verts = reinterpret_cast<double *>(ctx->swept.d_out.get());
    A.segs = reinterpret_cast<int *>(ctx->swept.d_out + o_segs);
    A.tris = reinterpret_cast<int *>(ctx->swept.d_out + o_tris);
    CK(launch_swept(4, A, st));
    CK(launch_swept(5, A, st));
    ctx->launches += 2;
    const SweptProblem &last = tab[n - 1];
    const size_t b_field = prm->want_field ? ((size_t)last.blk0 * kSweptBlock + (size_t)last.nx * last.ny) * 8 : 0;
    CK(ctx->h_stage.reserve(o_end + b_field + 16));
    unsigned char *hs = ctx->h_stage;
    if (o_end) CK(cudaMemcpyAsync(hs, ctx->swept.d_out, o_end, cudaMemcpyDeviceToHost, st));
    if (b_field) CK(cudaMemcpyAsync(hs + o_end, A.field, b_field, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    // every problem's arrays, as the single call allocates them; a problem with a non-finite value gets none
    int64_t v0 = 0, s0 = 0, f0 = 0;
    for (int k = 0; k < n; ++k) {
        const SweptProblem &g = tab[k];
        const int *ps = pst + 8 * k;
        const int64_t Vk = (int64_t)ps[2] + ps[3] + ps[4], Sk = ps[5], Fk = ps[6];
        const int64_t vk = v0, sk = s0, fk = f0;
        v0 += Vk; s0 += Sk; f0 += Fk;
        if (ps[0]) {
            status_out[k] = SVSDF_ERR_NONFINITE;
            continue;
        }
        svsdf_swept_mesh *o = &out[k];
        const size_t bf = prm->want_field ? (size_t)g.nx * g.ny * 8 : 0;
        o->vertices = static_cast<double *>(std::malloc((size_t)Vk * 16 + 16));
        o->segments = static_cast<int32_t *>(std::malloc((size_t)Sk * 8 + 16));
        o->triangles = static_cast<int32_t *>(std::malloc((size_t)Fk * 12 + 16));
        o->field = bf ? static_cast<double *>(std::malloc(bf)) : nullptr;
        if (!o->vertices || !o->segments || !o->triangles || (bf && !o->field)) {
            for (int j = 0; j <= k; ++j) {
                svsdf_swept_free(&out[j]);
                if (multi) status_out[j] = SVSDF_ERR_INVALID;
            }
            ctx->err = who + ": out of host memory";
            return SVSDF_ERR_INVALID;
        }
        o->i0 = g.i0; o->j0 = g.j0; o->nx = g.nx; o->ny = g.ny;
        o->n_vertices = Vk; o->n_segments = Sk; o->n_triangles = Fk;
        o->clipped = ps[1] ? 1 : 0;
        o->n_evaluated = ps[7];
        std::memcpy(o->vertices, hs + (size_t)vk * 16, (size_t)Vk * 16);
        std::memcpy(o->segments, hs + o_segs + (size_t)sk * 8, (size_t)Sk * 8);
        std::memcpy(o->triangles, hs + o_tris + (size_t)fk * 12, (size_t)Fk * 12);
        if (bf) std::memcpy(o->field, hs + o_end + (size_t)g.blk0 * kSweptBlock * 8, bf);
        if (multi) status_out[k] = SVSDF_OK;
    }
    return SVSDF_OK;
}
}  // namespace

int svsdf_swept_contour(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, const svsdf_swept_params *prm,
                        svsdf_swept_mesh *out) {
    if (!ctx || !prm || !out) return SVSDF_ERR_INVALID;
    std::memset(out, 0, sizeof(*out));
    const svsdf_clearance_problem p{N, T, coeffs};
    return swept_run(ctx, false, 1, &p, prm, out, nullptr);
}

int svsdf_swept_contour_multi(svsdf_ctx *ctx, int n, const svsdf_clearance_problem *problems, const svsdf_swept_params *params,
                              svsdf_swept_mesh *out, int *status_out) {
    if (!ctx) return SVSDF_ERR_INVALID;
    if (n < 0 || n > kMaxMultiProblems || !params || (n > 0 && (!problems || !out || !status_out))) {
        ctx->err = "svsdf_swept_contour_multi: needs 0 <= n <= 65535, the parameters and the problem, output and status arrays";
        return SVSDF_ERR_INVALID;
    }
    for (int k = 0; k < n; ++k) {
        std::memset(&out[k], 0, sizeof(out[k]));
        status_out[k] = SVSDF_ERR_INVALID;
    }
    return swept_run(ctx, true, n, problems, params, out, status_out);
}

void svsdf_swept_free(svsdf_swept_mesh *mesh) {
    if (!mesh) return;
    std::free(mesh->vertices);
    std::free(mesh->segments);
    std::free(mesh->triangles);
    std::free(mesh->field);
    mesh->vertices = nullptr;
    mesh->segments = nullptr;
    mesh->triangles = nullptr;
    mesh->field = nullptr;
}

// ---- svsdf_map_clearance (kernels: svsdf_clearance.cu; why the band is exact: DESIGN.md §7) -----------------------------------------
namespace {
void clearance_empty(svsdf_clearance *out) {
    std::memset(out, 0, sizeof(*out));
    out->min_sdf = INFINITY;
    out->argmin = -1;
}

// the band's samples: rho and the samples of svsdf_swept_contour with iso = d_max.  Returns `all` (every occupied column is in the band,
// no samples): d_max = +inf or a shape without a far-field bound.
bool clearance_samples(const svsdf_ctx *ctx, int N, const double *T, const double *coeffs, double D, double d_max, std::vector<double> &samp) {
    const ShapeParams &S = ctx->shape;
    samp.clear();
    if (!(S.rout < 1e299) || !std::isfinite(d_max)) return true;
    const double rho = std::max(std::max(S.prune_rmin, S.rout + S.prune_scale * d_max), 0.0);
    swept_samples(ctx, N, T, coeffs, D, rho, samp);
    return false;
}

// The list and summary of one trajectory from its band (P cells in map order: ij, centres, values, t*): the cells with value <= d_max.
int clearance_list(svsdf_ctx *ctx, int64_t P, const int32_t *h_ij, const double *h_xy, const double *h_sdf, const double *h_ts,
                   unsigned long long n_occ, double d_max, svsdf_clearance *out) {
    int64_t n_within = 0;
    for (int64_t p = 0; p < P; ++p) {
        if (!std::isfinite(h_sdf[p])) {
            ctx->err = "svsdf_map_clearance: non-finite value";
            return SVSDF_ERR_NONFINITE;
        }
        n_within += h_sdf[p] <= d_max;
    }
    out->ij = static_cast<int32_t *>(std::malloc((size_t)n_within * 8 + 16));
    out->xy = static_cast<double *>(std::malloc((size_t)n_within * 16 + 16));
    out->sdf = static_cast<double *>(std::malloc((size_t)n_within * 8 + 16));
    out->tstar = static_cast<double *>(std::malloc((size_t)n_within * 8 + 16));
    if (!out->ij || !out->xy || !out->sdf || !out->tstar) {
        svsdf_clearance_free(out);
        ctx->err = "svsdf_map_clearance: out of host memory";
        return SVSDF_ERR_INVALID;
    }
    int64_t k = 0, n_coll = 0;
    for (int64_t p = 0; p < P; ++p) {
        const double v = h_sdf[p];
        if (!(v <= d_max)) continue;
        out->ij[2 * k] = h_ij[2 * p];
        out->ij[2 * k + 1] = h_ij[2 * p + 1];
        out->xy[2 * k] = h_xy[2 * p];
        out->xy[2 * k + 1] = h_xy[2 * p + 1];
        out->sdf[k] = v;
        out->tstar[k] = h_ts[p];
        n_coll += v <= 0.0;
        if (v < out->min_sdf) {  // strict: the first in list order among ties
            out->min_sdf = v;
            out->argmin = k;
        }
        ++k;
    }
    out->n_occupied = (int64_t)n_occ;
    out->n_evaluated = P;
    out->n_within = n_within;
    out->n_colliding = n_coll;
    return SVSDF_OK;
}

// cell index range [lo, hi] of the map axis (n cells, origin o, resolution res) whose centres may lie in [a, b]: outward by one cell
// beyond the rounding of the centres, clipped to the map (lo > hi: none)
void cell_range(double a, double b, double o, double res, int n, int &lo, int &hi) {
    const double l = std::floor((a - o) / res - 0.5) - 1.0, h = std::ceil((b - o) / res - 0.5) + 1.0;  // a, b: not NaN, maybe infinite
    lo = (int)std::min(std::max(l, 0.0), (double)n);
    hi = (int)std::max(std::min(h, (double)n - 1.0), -1.0);
}

// The bands of n trajectories, built in one count / scan / write (DESIGN.md §7).  Problem k's band is cells off[k] .. off[k + 1] - 1
// of the concatenation in ctx->swept.d_cl_point: (i, j) int32 pairs at 0, then centres, values and t* at o_pts, o_sdf, o_ts (contiguous, so
// one download brings them all).
struct ClearanceBands {
    std::vector<int64_t> off;
    unsigned long long n_occ = 0;  // occupied columns of the map
    size_t o_pts = 0, o_sdf = 0, o_ts = 0, o_end = 0;
};

// The checks of svsdf_map_clearance[_multi] (`multi`: messages name the call and the problem), then the bands.  Nothing is launched
// for n = 0 or when a check fails.
int clearance_bands(svsdf_ctx *ctx, bool multi, int n, const svsdf_clearance_problem *problems, double d_max, ClearanceBands &B) {
    const std::string who = multi ? "svsdf_map_clearance_multi" : "svsdf_map_clearance";
    auto invalid = [&](const std::string &msg) {
        ctx->err = msg;
        return SVSDF_ERR_INVALID;
    };
    B.off.assign(n + 1, 0);
    // the band proves only "outer value > d_max"; for d_max >= 0 that value is the whole answer (no interior branch), below 0 it is not
    if (!(d_max >= 0.0)) return invalid(who + ": d_max must be >= 0 or +INFINITY");
    std::vector<double> dur(n);
    for (int k = 0; k < n; ++k) {
        const svsdf_clearance_problem &p = problems[k];
        const char *msg = nullptr;
        BlobLayout L;
        bool ok = traj_layout(p.N, p.T, p.coeffs, L, dur[k], &msg) == SVSDF_OK;
        for (int64_t e = 0; ok && e < 18 * (int64_t)p.N; ++e)
            if (!std::isfinite(p.coeffs[e])) {
                ok = false;
                msg = "svsdf_map_clearance: non-finite trajectory coefficient";
            }
        if (!ok) return invalid(multi ? who + ": problem " + std::to_string(k) + ": " + msg : std::string(msg));
    }
    if (n == 0) return SVSDF_OK;
    if (!ctx->map()) {
        ctx->err = who + ": map not set";
        return SVSDF_ERR_NOT_READY;
    }
    if ((int64_t)ctx->map_X * ctx->map_Y > 2000000000LL) return invalid(who + ": map has more than 2e9 columns");
    ClearanceArgs A;
    std::memset(&A, 0, sizeof(A));
    A.map = ctx->map();
    A.X = ctx->map_X; A.Y = ctx->map_Y; A.h = ctx->map_h; A.row_bytes = ctx->map_row_bytes; A.Z = ctx->map_Z;
    A.layer = (int64_t)(A.X + 2 * A.h) * A.row_bytes;
    A.ox = ctx->map_ox; A.oy = ctx->map_oy; A.res = ctx->map_res;
    // per problem: its samples and its reach rectangle (the bounding box of the samples' discs, padded outwards by a relative margin far
    // above the rounding of the kernel's test dx*dx + dy*dy <= r*r, then by one cell; clipped to the map), padded to whole CTAs
    std::vector<ClearanceProblem> cp(n + 1);
    std::vector<double> samp_all, samp;
    int64_t cta = 0, cells = 0;
    for (int k = 0; k <= n; ++k) {
        ClearanceProblem &c = cp[k];
        std::memset(&c, 0, sizeof(c));
        c.cta0 = cta;
        int i0 = 0, i1 = A.X - 1, j0 = 0, j1 = A.Y - 1;
        if (k == n) {
            c.all = c.occ_only = 1;
        } else {
            const svsdf_clearance_problem &p = problems[k];
            c.all = clearance_samples(ctx, p.N, p.T, p.coeffs, dur[k], d_max, samp) ? 1 : 0;
            c.n_samp = (int)(samp.size() / 3);
            if (c.n_samp > kSweptMaxSamples) return invalid(who + ": too many path samples");
            c.samp0 = (int)(samp_all.size() / 3);
            samp_all.insert(samp_all.end(), samp.begin(), samp.end());
            if (!c.all) {
                double x0 = INFINITY, x1 = -INFINITY, y0 = INFINITY, y1 = -INFINITY;
                for (int s = 0; s < c.n_samp; ++s) {
                    const double sx = samp[3 * s], sy = samp[3 * s + 1], r = samp[3 * s + 2];
                    const double m = r + 1e-9 * (std::fabs(sx) + std::fabs(sy) + r + 1.0);
                    x0 = std::min(x0, sx - m); x1 = std::max(x1, sx + m);
                    y0 = std::min(y0, sy - m); y1 = std::max(y1, sy + m);
                }
                cell_range(x0, x1, A.ox, A.res, A.X, i0, i1);
                cell_range(y0, y1, A.oy, A.res, A.Y, j0, j1);
            }
        }
        if (i0 <= i1 && j0 <= j1) {
            c.i0 = i0;
            c.wy0 = (j0 + A.h) / 32;
            c.nW = (j1 + A.h) / 32 - c.wy0 + 1;
            c.n_items = (int64_t)(i1 - i0 + 1) * c.nW;
            // the map cells its words hold (its band is a subset of them): its rows times the map columns y0 .. y1 - 1 of its words
            const int64_t y0 = std::max(32 * (int64_t)c.wy0 - A.h, (int64_t)0), y1 = std::min(32 * (int64_t)(c.wy0 + c.nW) - A.h, (int64_t)A.Y);
            if (k < n) cells += (int64_t)(i1 - i0 + 1) * (y1 - y0);
        } else {
            c.nW = 1;
        }
        cta += (c.n_items + 255) / 256;
    }
    // Band positions, the per-CTA prefix (k_sw_scan) and the band total are int32, and so are the CTA indices (grid x dimension).  The
    // map cells of the rectangles' words bound the band total; one problem holds at most X Y <= 2e9 of them, so a single trajectory
    // is never refused here.  A problem's words are no more than its cells, so its CTAs number at most cells / 256 + 1.
    if (cells > 2147483647LL || cta > 2147483647LL)
        return invalid(who + ": the problems' rectangles hold more than 2^31 - 1 cells");
    CK(cudaSetDevice(ctx->device));
    const int nblk = (int)cta;
    A.n_items = (int64_t)nblk * 256;
    A.n_prob = n + 1;
    // small: header [0] occupied columns (u64), [8] band cells (int) | per-CTA counts | problem table | samples
    const size_t off_blk = 64, off_prob = align16(off_blk + (size_t)(nblk + 1) * 4), off_samp = align16(off_prob + cp.size() * sizeof(ClearanceProblem)),
                 small = off_samp + samp_all.size() * 8;
    CK(ctx->swept.d_cl_small.reserve(small));
    CK(ctx->swept.d_cl_band.reserve((size_t)A.n_items * 4));
    CK(ctx->h_stage.reserve(small));
    unsigned char *hs = ctx->h_stage;
    std::memset(hs, 0, off_prob);
    std::memcpy(hs + off_prob, cp.data(), cp.size() * sizeof(ClearanceProblem));
    if (!samp_all.empty()) std::memcpy(hs + off_samp, samp_all.data(), samp_all.size() * 8);
    A.n_occ = reinterpret_cast<unsigned long long *>(ctx->swept.d_cl_small.get());
    A.blk = reinterpret_cast<int *>(ctx->swept.d_cl_small + off_blk);
    A.prob = reinterpret_cast<const ClearanceProblem *>(ctx->swept.d_cl_small + off_prob);
    A.samp = reinterpret_cast<const double *>(ctx->swept.d_cl_small + off_samp);
    A.band = reinterpret_cast<unsigned *>(ctx->swept.d_cl_band.get());
    cudaStream_t st = ctx->stream;
    CK(cudaMemcpyAsync(ctx->swept.d_cl_small, hs, small, cudaMemcpyHostToDevice, st));
    CK(launch_clearance(0, A, st));
    CK(launch_swept_scan(A.blk, nblk, 1, reinterpret_cast<int *>(ctx->swept.d_cl_small + 8), st));
    CK(cudaMemcpyAsync(hs, ctx->swept.d_cl_small, off_prob, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    ctx->launches += 2;
    std::memcpy(&B.n_occ, hs, 8);
    for (int k = 0; k <= n; ++k) B.off[k] = reinterpret_cast<const int *>(hs + off_blk)[cp[k].cta0];
    const int64_t P = B.off[n];
    B.o_pts = align16((size_t)P * 8);
    B.o_sdf = B.o_pts + (size_t)P * 16;
    B.o_ts = B.o_sdf + (size_t)P * 8;
    B.o_end = B.o_ts + (size_t)P * 8;
    if (P > 0) {
        CK(ctx->swept.d_cl_point.reserve(B.o_end + 16));
        A.ij = reinterpret_cast<int *>(ctx->swept.d_cl_point.get());
        A.pts = reinterpret_cast<double *>(ctx->swept.d_cl_point + B.o_pts);
        CK(launch_clearance(1, A, st));
        ctx->launches += 1;
    }
    return SVSDF_OK;
}

// the band cells (all problems) with their values and t*, from the device into the host stage
int clearance_download(svsdf_ctx *ctx, const ClearanceBands &B) {
    CK(ctx->h_stage.reserve(B.o_end));
    CK(cudaMemcpyAsync(ctx->h_stage, ctx->swept.d_cl_point, B.o_end, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return SVSDF_OK;
}

// the list and summary of problem k from the host stage
int clearance_out(svsdf_ctx *ctx, const ClearanceBands &B, int k, double d_max, svsdf_clearance *out) {
    const unsigned char *hs = ctx->h_stage;
    const int64_t o = B.off[k];
    return clearance_list(ctx, B.off[k + 1] - o, reinterpret_cast<const int32_t *>(hs) + 2 * o, reinterpret_cast<const double *>(hs + B.o_pts) + 2 * o,
                          reinterpret_cast<const double *>(hs + B.o_sdf) + o, reinterpret_cast<const double *>(hs + B.o_ts) + o, B.n_occ, d_max, out);
}
}  // namespace

int svsdf_map_clearance(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, double d_max, svsdf_clearance *out) {
    if (!ctx || !out) return SVSDF_ERR_INVALID;
    clearance_empty(out);
    const svsdf_clearance_problem p{N, T, coeffs};
    ClearanceBands B;
    int rc = clearance_bands(ctx, false, 1, &p, d_max, B);
    if (rc) return rc;
    const int64_t P = B.off[1];
    if (P > 0) {
        // svsdf_query's path (outer solve, then the interior branch) on the band: the same kernels, so the same bits per point
        rc = upload_traj(ctx, N, T, coeffs, P);
        if (rc) return rc;
        double *pts = reinterpret_cast<double *>(ctx->swept.d_cl_point + B.o_pts);
        rc = run_kernels(ctx, pts, P, false, true, reinterpret_cast<double *>(ctx->swept.d_cl_point + B.o_sdf),
                         reinterpret_cast<double *>(ctx->swept.d_cl_point + B.o_ts), nullptr, nullptr);
        if (rc) return rc;
        rc = clearance_download(ctx, B);
        if (rc) return rc;
    }
    return clearance_out(ctx, B, 0, d_max, out);
}

// The bands of all problems in one count / scan / write, then one multi-problem evaluation of the concatenated bands (DESIGN.md §7).
int svsdf_map_clearance_multi(svsdf_ctx *ctx, int n, const svsdf_clearance_problem *problems, double d_max, svsdf_clearance *out,
                              int *status_out) {
    if (!ctx) return SVSDF_ERR_INVALID;
    if (n < 0 || n > kMaxMultiProblems || (n > 0 && (!problems || !out || !status_out))) {
        ctx->err = "svsdf_map_clearance_multi: needs 0 <= n <= 65535 and the problem, output and status arrays";
        return SVSDF_ERR_INVALID;
    }
    for (int k = 0; k < n; ++k) {
        clearance_empty(&out[k]);
        status_out[k] = SVSDF_ERR_INVALID;
    }
    ClearanceBands B;
    int rc = clearance_bands(ctx, true, n, problems, d_max, B);
    if (rc || n == 0) return rc;
    if (B.off[n] > 0) {
        // the problems with a band, in problem order: their points are the concatenation's, in the same order
        std::vector<MultiItem> items;
        for (int k = 0; k < n; ++k) {
            if (B.off[k + 1] == B.off[k]) continue;
            MultiItem it;
            it.N = problems[k].N; it.T = problems[k].T; it.coeffs = problems[k].coeffs; it.P = B.off[k + 1] - B.off[k];
            items.push_back(it);
        }
        const PointQuery pq{reinterpret_cast<double *>(ctx->swept.d_cl_point + B.o_pts), reinterpret_cast<double *>(ctx->swept.d_cl_point + B.o_sdf),
                            reinterpret_cast<double *>(ctx->swept.d_cl_point + B.o_ts)};
        rc = run_multi(ctx, items.data(), (int)items.size(), nullptr, &pq);
        if (rc) return rc;
        for (const MultiItem &it : items)
            if (it.rc != SVSDF_OK) {
                ctx->err = "svsdf_map_clearance_multi: a problem was refused by the evaluation";
                return SVSDF_ERR_INVALID;
            }
        rc = clearance_download(ctx, B);
        if (rc) return rc;
    }
    for (int k = 0; k < n; ++k) status_out[k] = clearance_out(ctx, B, k, d_max, &out[k]);
    return SVSDF_OK;
}

void svsdf_clearance_free(svsdf_clearance *c) {
    if (!c) return;
    std::free(c->ij);
    std::free(c->xy);
    std::free(c->sdf);
    std::free(c->tstar);
    c->ij = nullptr;
    c->xy = nullptr;
    c->sdf = nullptr;
    c->tstar = nullptr;
}

}  // extern "C"
