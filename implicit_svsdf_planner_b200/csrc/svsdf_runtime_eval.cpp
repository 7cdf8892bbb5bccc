// svsdf_runtime_eval.cpp — the single-problem evaluation: trajectory blob, pose table, the k_outer / k_gsip launch plan and the
// cost, gradient and query entry points (svsdf_cost_grad, svsdf_evaluate: the path bench.py times).  Nothing on that path leaves
// this unit.
#include <algorithm>
#include <cmath>

#include "svsdf_runtime.h"

int ensure_scratch(svsdf_ctx *ctx, int64_t P) {
    CK(ctx->d_flag.reserve(P));
    CK(ctx->d_inside_tstar.reserve(P));
    CK(ctx->d_inside_list.reserve(P));
    CK(ctx->d_gsip_contrib.reserve((size_t)P * 20));
    CK(ctx->d_gsip_piece.reserve(P));
    return SVSDF_OK;
}

namespace {

// Which pose windows the evaluation of P points builds (0 / 1 / 2: none / layer 2 / layers 2 and 3).  The layer-2 windows are
// always cheap: (K1 + 1) x 21 records, at most 42 k at D < 300 s.  The layer-3 windows hold (K1 + 1) x 22 x 21 records (0.9 M, 30 MB
// at D near 300 s) and each replaces one trajectory evaluation of one point's layer-3 scan (21 per point): they are built when they
// hold at most kWin3PerSample records per sample they serve.  Measured on an H100 (scripts/pose_windows_sweep.py, strict build):
// they still pay at 3.0 records per sample (K1 = 134, P = 1 000: 3 % off the evaluation) and at 1.8 (K1 = 1999, P = 25 000: 1.5 %).
constexpr int64_t kWin3PerSample = 2;
int pose_windows(const svsdf_ctx *ctx, int K1, int64_t P) {
    if (ctx->hooks.force_pose_windows >= 0) return std::min(ctx->hooks.force_pose_windows, 2);  // test hook
    return win3_records(K1) <= kWin3PerSample * kWinLen * P ? 2 : 1;
}

// The layer-1 pose table of the uploaded blob and the pose windows for an evaluation of P points, in one launch.
int pose_table(svsdf_ctx *ctx, int64_t P) {
    const int K1 = ctx->layout.K1;
    ctx->win_layers = 0;  // a failed reserve leaves no windows to read
    const int layers = pose_windows(ctx, K1, P);
    if (layers > 0) CK(ctx->d_win.reserve(win2_records(K1) + (layers > 1 ? win3_records(K1) : 0)));
    PoseRec *w2 = layers > 0 ? ctx->d_win.get() : nullptr, *w3 = layers > 1 ? ctx->d_win + win2_records(K1) : nullptr;
    CK(kernels(ctx).pose_table(ctx->d_blob, K1, w2, w3, ctx->stream));
    ctx->win_layers = layers;
    ctx->launches += 1;
    return SVSDF_OK;
}

}  // namespace

int traj_layout(int N, const double *T, const double *coeffs, BlobLayout &L, double &D, const char **err) {
    if (N < 1 || N > kMaxPieces || !T || !coeffs) {
        *err = "svsdf: N out of range (1..64) or null trajectory";
        return SVSDF_ERR_INVALID;
    }
    D = 0.0;  // Trajectory::getTotalDuration (trajectory.hpp:410-419)
    for (int i = 0; i < N; ++i) {
        if (!(T[i] > 0.0) || !std::isfinite(T[i])) {
            *err = "svsdf: non-positive or non-finite piece duration";
            return SVSDF_ERR_INVALID;
        }
        D += T[i];
    }
    if (!(D < kMaxDuration)) {
        // The reference silently keeps the previous duration in this case (sw_manager.hpp:380); we refuse.
        *err = "svsdf: total duration >= 300 s is not supported (reference updateTraj ignores it)";
        return SVSDF_ERR_INVALID;
    }
    // layer-1 lattice: for (t = 0; t <= D; t += 0.15)
    int K1 = 0;
    for (double t = 0.0; t <= D; t += 0.15) K1++;
    L = blob_layout(N, K1);
    return SVSDF_OK;
}

void fill_blob(double *h, const BlobLayout &L, const double *T, const double *coeffs, double D) {
    const int N = L.N;
    std::memset(h, 0, (size_t)L.off_pose * sizeof(double));
    h[0] = (double)N;
    h[1] = (double)L.K1;
    h[2] = D;
    for (int i = 0; i < N; ++i) h[L.off_T + i] = T[i];
    // coefficients: MINCO b (col-major 6N x 3) -> [piece][dim][power]  (minco.hpp:515-528 builds the same
    // per-piece matrices, stored there highest power first)
    for (int i = 0; i < N; ++i)
        for (int d = 0; d < 3; ++d)
            for (int k = 0; k < 6; ++k) h[L.off_c + 18 * i + 6 * d + k] = coeffs[(size_t)d * 6 * N + 6 * i + k];
    {
        int k = 0;
        for (double t = 0.0; t <= D; t += 0.15) h[L.off_lat + k++] = t;
    }
}

int upload_traj(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, int64_t P, bool launch_pose) {
    BlobLayout L;
    double D = 0.0;
    const char *msg = nullptr;
    if (traj_layout(N, T, coeffs, L, D, &msg) != SVSDF_OK) {
        ctx->err = msg;
        return SVSDF_ERR_INVALID;
    }
    CK(ctx->h_blob.reserve(L.total));
    CK(ctx->d_blob.reserve(L.total));
    double *h = ctx->h_blob;
    fill_blob(h, L, T, coeffs, D);
    CK(cudaMemcpyAsync(ctx->d_blob, h, (size_t)L.off_pose * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    ctx->layout = L;
    ctx->traj_N = N;
    ctx->traj_D = D;
    if (launch_pose) return pose_table(ctx, P);
    return SVSDF_OK;
}

// Resident CTAs per SM of the single-problem k_outer and k_gsip for a trajectory of N pieces and `blob` doubles: the grids are sized
// as SMs x occupancy so that the warp-stride loops run as exactly one full wave (no partial second wave).
int occupancy(svsdf_ctx *ctx, int N, int blob, Occupancy *occ) {
    const auto key = std::make_tuple(N, blob, ctx->scaled ? 1 : 0);
    auto it = ctx->occ_cache.find(key);
    if (it == ctx->occ_cache.end()) {
        int oo = 0, og = 0, ch = 1;
        CK(kernels(ctx).query_occupancy(ctx->shape, N, blob, &oo, &og, &ch));
        it = ctx->occ_cache.emplace(key, Occupancy{oo > 0 ? oo : 1, og > 0 ? og : 1, ch}).first;
    }
    *occ = it->second;
    return SVSDF_OK;
}

// k_outer's launch for P points, shared by svsdf_cost_grad and every problem of svsdf_cost_grad_multi (which is what gives a multi
// problem the bits of its single call).  One warp per point, 8 warps per CTA, warp-stride loop; the grid is at most one full wave.
// The batched schedule pays off once every warp owns a couple of dozen points; small problems keep one point per warp.
OuterPlan outer_plan(const svsdf_ctx *ctx, int64_t P, const Occupancy &occ) {
    int64_t need = (P + kWarpsPerBlock - 1) / kWarpsPerBlock;
    const int64_t cap = (int64_t)ctx->sm_count * occ.outer;
    if (need < 1) need = 1;
    OuterPlan plan;
    plan.grid = (int)(need < cap ? need : cap);
    if (ctx->hooks.force_grid_outer > 0) plan.grid = ctx->hooks.force_grid_outer;  // test hook
    plan.batched = (P >= (int64_t)16 * plan.grid * kWarpsPerBlock) ? 1 : 0;
    if (ctx->hooks.force_batched >= 0) plan.batched = ctx->hooks.force_batched;  // test hook
    return plan;
}

// Batches of a warp per descent pass of a batched k_outer launch whose warps own up to `rounds` batches and whose shared memory is
// sized by (blob, N): as many as there are rounds, up to what keeps the residency (occ.chunk).  The chunk changes who solves a point
// and when, never a bit of the results, so a problem's may differ between its single and its multi call.
int outer_chunk(const svsdf_ctx *ctx, const Occupancy &occ, int64_t rounds, int blob, int N) {
    int64_t c = std::min<int64_t>(occ.chunk, rounds);
    if (ctx->hooks.force_outer_chunk > 0) c = std::min(ctx->hooks.force_outer_chunk, kOuterChunkMax);  // test hook
    while (c > 1 && outer_smem_doubles(blob, N, (int)c) * sizeof(double) > kMaxDynSmemBytes) --c;
    return (int)std::max<int64_t>(c, 1);
}
int64_t outer_rounds(int64_t P, int grid) {
    const int64_t per = (int64_t)32 * grid * kWarpsPerBlock;
    return (P + per - 1) / per;
}

// k_gsip's variant from the interior points of the previous evaluation (-1: none): few -> 22-warp CTAs (one warp per ring sample,
// lower latency; the variant does not change the bits, tests/test_gpu_gsip.py).  grid: the test hook's, or 0 for one full wave.
GsipPlan gsip_plan(const svsdf_ctx *ctx, int64_t prev_inside) {
    GsipPlan plan;
    plan.wide = (prev_inside >= 0 && prev_inside <= ctx->sm_count) ? 1 : 0;
    if (ctx->hooks.force_gsip_wide >= 0) plan.wide = ctx->hooks.force_gsip_wide ? 1 : 0;  // test hook
    plan.grid = ctx->hooks.force_grid_gsip > 0 ? ctx->hooks.force_grid_gsip : 0;        // test hook
    return plan;
}

int run_kernels(svsdf_ctx *ctx, const double *d_points, int64_t P, bool reduce, bool gsip, double *o_sdf,
                double *o_ts, double *o_grad, int *o_rounds) {
    const int N = ctx->traj_N;
    int rc = ensure_scratch(ctx, P);
    if (rc) return rc;
    Occupancy occ;
    rc = occupancy(ctx, N, ctx->layout.total, &occ);
    if (rc) return rc;
    const OuterPlan plan = outer_plan(ctx, P, occ);
    const int grid = plan.grid;
    const int nacc = 19 * N + 1;
    if (reduce) {
        CK(ctx->d_partials.reserve((size_t)grid * nacc));
        CK(ctx->d_out.reserve(nacc + 1));
        CK(ctx->d_tot.reserve(nacc + 1));
        CK(ctx->h_out.reserve(nacc + 1));
    }
    KernelArgs A;
    std::memset(&A, 0, sizeof(A));
    A.blob = ctx->d_blob;
    A.blob_doubles = ctx->layout.total;
    A.points_xy = d_points;
    A.P = P;
    A.cp = ctx->cp;
    A.out_sdf = o_sdf; A.out_tstar = o_ts; A.out_grad = o_grad; A.out_rounds = o_rounds;
    A.partials = ctx->d_partials;
    A.want_reduce = reduce ? 1 : 0;
    A.want_gsip = gsip ? 1 : 0;
    A.batched = plan.batched;
    A.outer_chunk = outer_chunk(ctx, occ, outer_rounds(P, grid), A.blob_doubles, N);
    A.inside_flag = ctx->d_flag;
    A.inside_tstar = ctx->d_inside_tstar;
    A.inside_list = ctx->d_inside_list;
    A.n_inside = ctx->d_n_inside;
    A.gsip_contrib = ctx->d_gsip_contrib;
    A.gsip_piece = ctx->d_gsip_piece;
    A.eval_counter = ctx->count_evals ? ctx->d_eval_counter.get() : nullptr;
    A.win2 = ctx->win_layers > 0 ? ctx->d_win.get() : nullptr;
    A.win3 = ctx->win_layers > 1 ? ctx->d_win + win2_records(ctx->layout.K1) : nullptr;
    GsipPlan gp = gsip_plan(ctx, reduce ? ctx->last_n_inside : -1);
    if (gp.grid == 0) gp.grid = gp.wide ? ctx->sm_count : ctx->sm_count * occ.gsip;
    if (!gsip) CK(cudaMemsetAsync(ctx->d_n_inside, 0, sizeof(int), ctx->stream));
    size_t smem = outer_smem_doubles(A.blob_doubles, N, 1) * sizeof(double);
    if (smem > kMaxDynSmemBytes) {
        ctx->err = "svsdf: trajectory blob does not fit in shared memory";
        return SVSDF_ERR_INVALID;
    }
    cudaEvent_t mark = ctx->mark_kernels ? ctx->evk[2] : nullptr;
    const Kernels &K = kernels(ctx);
    CK(K.cost_kernels(A, ctx->shape, ctx->scaled ? &ctx->sched : nullptr, N, grid, gp.grid, ctx->stream, mark, gp.wide));
    ctx->launches += gsip ? 3 : 1;
    if (ctx->mark_kernels) CK(cudaEventRecord(ctx->evk[3], ctx->stream));
    if (reduce) {
        CK(K.finalize(ctx->d_partials, grid, N, ctx->d_n_inside, ctx->d_gsip_contrib, ctx->d_gsip_piece, ctx->d_tot, ctx->d_ticket,
                      ctx->d_out, ctx->stream));
        ctx->launches += 1;
    }
    return SVSDF_OK;
}

int pose_ready(svsdf_ctx *ctx, const char *who) {
    if (!ctx->pose_on || (ctx->map3d && ctx->map())) return SVSDF_OK;
    ctx->err = std::string(who) + ": the pose penalty needs a 3-D map (svsdf_set_map3d)";
    return SVSDF_ERR_NOT_READY;
}

int launch_pose(svsdf_ctx *ctx, const host::PoseParams &pp, const double *half, const double *blobs, const PoseProblem *prob, int n,
                int max_N, double *rec) {
    PoseArgs A;
    std::memset(&A, 0, sizeof(A));
    A.map = ctx->map();
    A.X = ctx->map_X; A.Y = ctx->map_Y; A.Z = ctx->map_Z; A.h = ctx->map_h; A.row_bytes = ctx->map_row_bytes;
    A.layer = (int64_t)(A.X + 2 * A.h) * A.row_bytes;
    A.res = ctx->map_res;
    const double lo[3] = {ctx->map_ox, ctx->map_oy, ctx->map_oz};
    const int size[3] = {A.X, A.Y, A.Z};
    for (int a = 0; a < 3; ++a) {
        A.lo[a] = lo[a];
        A.hi[a] = lo[a] + (double)size[a] * A.res;  // boundary_xyzmax as extract_impl takes it
        A.half[a] = half[a];
    }
    A.safety_hor = ctx->cp.safety_hor;
    A.res_samples = pp.res;
    A.n = n;
    A.blobs = blobs;
    A.prob = prob;
    A.rec = rec;
    CK(kernels(ctx).pose(A, ctx->shape, max_N * (pp.res + 1), ctx->stream));
    ctx->launches += 1;
    return SVSDF_OK;
}

namespace {

// R1 on the context's points; result (1 + 19N + 1 doubles) lands in ctx->h_out after the stream sync.  pose: also the pose penalty's
// sample records, right behind it in h_out (the same download).
int cost_grad_raw(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, bool pose = false) {
    if (!ctx->points() || ctx->P < 0) {
        ctx->err = "svsdf: query points not set";
        return SVSDF_ERR_NOT_READY;
    }
    int rc = upload_traj(ctx, N, T, coeffs, ctx->P);
    if (rc) return rc;
    const int nout = 1 + 19 * N + 1;
    const int npose = pose ? 4 * N * (ctx->pose.res + 1) : 0;
    if (ctx->time_kernels) CK(cudaEventRecord(ctx->ev0, ctx->stream));
    if (pose) {
        CK(ctx->d_out.reserve(nout + npose));
        CK(ctx->h_out.reserve(nout + npose));
        rc = launch_pose(ctx, ctx->pose, ctx->pose_half, ctx->d_blob, nullptr, 1, N, ctx->d_out + nout);
        if (rc) return rc;
    }
    rc = run_kernels(ctx, ctx->points(), ctx->P, true, true, nullptr, nullptr, nullptr, nullptr);
    if (rc) return rc;
    if (ctx->time_kernels) CK(cudaEventRecord(ctx->ev1, ctx->stream));
    CK(cudaMemcpyAsync(ctx->h_out, ctx->d_out, (size_t)(nout + npose) * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (ctx->time_kernels) {
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
        ctx->gpu_ms_total += ms;
    }
    ctx->last_n_inside = (int64_t)ctx->h_out[1 + 19 * N];
    return SVSDF_OK;
}

double evaluate_impl(svsdf_ctx *ctx, const double *x, double *g, int n) {
    const int N = ctx->he.N;
    if (!ctx->have_boundary || n != N + 3 * (N - 1)) {
        ctx->err = "svsdf_evaluate: boundary conditions not set or wrong n";
        ctx->last_status = SVSDF_ERR_NOT_READY;
        return NAN;
    }
    int rc = pose_ready(ctx, "svsdf_evaluate");
    if (rc) {
        ctx->last_status = rc;
        return NAN;
    }
    ctx->n_evaluate++;
    ctx->he.forward(x);
    rc = cost_grad_raw(ctx, N, ctx->he.times.data(), ctx->he.minco.getCoeffs(), ctx->pose_on);
    if (rc) {
        ctx->last_status = rc;
        return NAN;
    }
    const double cost = ctx->he.backward(ctx->h_out, x, ctx->rho, ctx->pose_penalty(), ctx->h_out + (1 + 19 * N + 1), ctx->dynamics(), g,
                                         &ctx->cost_pos, &ctx->cost_other);
    ctx->cost_total = cost;
    ctx->last_status = SVSDF_OK;
    return cost;
}

}  // namespace

extern "C" {

int svsdf_set_traj(svsdf_ctx *ctx, int N, const double *T, const double *coeffs) {
    if (!ctx) return SVSDF_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    int rc = upload_traj(ctx, N, T, coeffs, ctx->P);
    if (rc) return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    return SVSDF_OK;
}

int svsdf_query(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, int64_t P, const double *pts,
                double *sdf, double *tstar, double *grad3, int *rounds, int outer_only) {
    if (!ctx || P < 0 || (P > 0 && !pts)) return SVSDF_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    int rc = upload_traj(ctx, N, T, coeffs, P);
    if (rc) return rc;
    if (P == 0) { CK(cudaStreamSynchronize(ctx->stream)); return SVSDF_OK; }
    CK(ctx->query.d_points.reserve((size_t)P * 2));
    CK(ctx->query.d_sdf.reserve(P));
    CK(ctx->query.d_ts.reserve(P));
    CK(ctx->query.d_grad.reserve((size_t)P * 3));
    CK(ctx->query.d_rounds.reserve(P));
    CK(ctx->h_stage.reserve((size_t)P * 5 * sizeof(double) + (size_t)P * sizeof(int)));
    double *h = reinterpret_cast<double *>(ctx->h_stage.get());
    pack_xy(h, pts, P, 3);
    CK(cudaMemcpyAsync(ctx->query.d_points, h, (size_t)P * 2 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    rc = run_kernels(ctx, ctx->query.d_points, P, false, outer_only == 0, ctx->query.d_sdf, ctx->query.d_ts, ctx->query.d_grad,
                     ctx->query.d_rounds);
    if (rc) return rc;
    double *h_sdf = h, *h_ts = h + P, *h_grad = h + 2 * P;
    int *h_rounds = reinterpret_cast<int *>(h + 5 * P);
    CK(cudaMemcpyAsync(h_sdf, ctx->query.d_sdf, (size_t)P * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(h_ts, ctx->query.d_ts, (size_t)P * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(h_grad, ctx->query.d_grad, (size_t)P * 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(h_rounds, ctx->query.d_rounds, (size_t)P * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (sdf) std::memcpy(sdf, h_sdf, (size_t)P * sizeof(double));
    if (tstar) std::memcpy(tstar, h_ts, (size_t)P * sizeof(double));
    if (grad3) std::memcpy(grad3, h_grad, (size_t)P * 3 * sizeof(double));
    if (rounds) std::memcpy(rounds, h_rounds, (size_t)P * sizeof(int));
    return SVSDF_OK;
}

int svsdf_cost_grad(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, double *cost_io,
                    double *gradT_io, double *gradC_io) {
    if (!ctx || !cost_io || !gradT_io || !gradC_io) return SVSDF_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    int rc = cost_grad_raw(ctx, N, T, coeffs);
    if (rc) return rc;
    const double *o = ctx->h_out;
    *cost_io += o[0];
    for (int e = 0; e < 18 * N; ++e) gradC_io[e] += o[1 + e];
    for (int i = 0; i < N; ++i) gradT_io[i] += o[1 + 18 * N + i];
    if (!std::isfinite(o[0])) return SVSDF_ERR_NONFINITE;
    return SVSDF_OK;
}

int svsdf_cost_grad_device(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, int repeats,
                           float *ms_per_eval, double *out_host) {
    if (!ctx || repeats < 1) return SVSDF_ERR_INVALID;
    if (!ctx->points()) { ctx->err = "svsdf: query points not set"; return SVSDF_ERR_NOT_READY; }
    CK(cudaSetDevice(ctx->device));
    int rc = upload_traj(ctx, N, T, coeffs, ctx->P, false);
    if (rc) return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaEventRecord(ctx->ev0, ctx->stream));
    for (int r = 0; r < repeats; ++r) {
        ctx->mark_kernels = (r == repeats - 1);
        if (ctx->mark_kernels) CK(cudaEventRecord(ctx->evk[0], ctx->stream));
        rc = pose_table(ctx, ctx->P);
        if (rc) return rc;
        if (ctx->mark_kernels) CK(cudaEventRecord(ctx->evk[1], ctx->stream));
        rc = run_kernels(ctx, ctx->points(), ctx->P, true, true, nullptr, nullptr, nullptr, nullptr);
        if (ctx->mark_kernels) cudaEventRecord(ctx->evk[4], ctx->stream);
        ctx->mark_kernels = false;
        if (rc) return rc;
    }
    CK(cudaEventRecord(ctx->ev1, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
    for (int k = 0; k < 4; ++k) CK(cudaEventElapsedTime(&ctx->last_kernel_ms[k], ctx->evk[k], ctx->evk[k + 1]));
    if (ms_per_eval) *ms_per_eval = ms / repeats;
    {
        const int nout = 1 + 19 * N + 1;
        CK(cudaMemcpy(ctx->h_out, ctx->d_out, (size_t)nout * sizeof(double), cudaMemcpyDeviceToHost));
        ctx->last_n_inside = (int64_t)ctx->h_out[1 + 19 * N];
        if (out_host) std::memcpy(out_host, ctx->h_out, (size_t)nout * sizeof(double));
    }
    return SVSDF_OK;
}

int svsdf_set_boundary(svsdf_ctx *ctx, const double *initS, const double *finalS, int N) {
    if (!ctx || !initS || !finalS || N < 2 || N > kMaxPieces) return SVSDF_ERR_INVALID;
    ctx->he.setup(initS, finalS, N);
    ctx->have_boundary = true;
    return SVSDF_OK;
}

double svsdf_evaluate(void *instance, const double *x, double *g, const int n) {
    svsdf_ctx *ctx = static_cast<svsdf_ctx *>(instance);
    if (!ctx || !x || !g) return NAN;
    if (cudaSetDevice(ctx->device) != cudaSuccess) return NAN;
    return evaluate_impl(ctx, x, g, n);
}

int svsdf_last_costs(const svsdf_ctx *ctx, double *out3) {
    if (!ctx || !out3) return SVSDF_ERR_INVALID;
    out3[0] = ctx->cost_pos; out3[1] = ctx->cost_other; out3[2] = ctx->cost_total;
    return SVSDF_OK;
}

int svsdf_get_traj(const svsdf_ctx *ctx, double *T_out, double *coeffs_out) {
    if (!ctx || !ctx->have_boundary) return SVSDF_ERR_NOT_READY;
    if (T_out) std::memcpy(T_out, ctx->he.times.data(), sizeof(double) * ctx->he.N);
    if (coeffs_out) std::memcpy(coeffs_out, ctx->he.minco.getCoeffs(), sizeof(double) * 18 * ctx->he.N);
    return SVSDF_OK;
}

int svsdf_pose_penalty_eval(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, const svsdf_pose_penalty *p, double *cost,
                            double *gradC, double *gradT, double *samples_out) {
    if (!ctx || !p || !cost || !gradC || !gradT) return SVSDF_ERR_INVALID;
    if (const int rc = pose_penalty_check(ctx, *p, "svsdf_pose_penalty_eval")) return rc;
    if (!ctx->map3d || !ctx->map()) {
        ctx->err = "svsdf_pose_penalty_eval: needs a 3-D map (svsdf_set_map3d)";
        return SVSDF_ERR_NOT_READY;
    }
    CK(cudaSetDevice(ctx->device));
    int rc = upload_traj(ctx, N, T, coeffs, 0, false);
    if (rc) return rc;
    host::PoseParams pp;
    pp.weight = p->weight;
    pp.res = p->integralIntervs;
    const size_t nrec = (size_t)4 * N * (pp.res + 1);
    CK(ctx->d_pose_rec.reserve(nrec));
    rc = launch_pose(ctx, pp, p->half, ctx->d_blob, nullptr, 1, N, ctx->d_pose_rec);
    if (rc) return rc;
    std::vector<double> rec(nrec), gc((size_t)18 * N, 0.0), gt(N, 0.0), partial(N, 0.0);
    CK(cudaMemcpyAsync(rec.data(), ctx->d_pose_rec, nrec * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    *cost = host::pose_penalty(pp, N, T, coeffs, rec.data(), gc.data(), gt.data(), partial.data());
    std::memcpy(gradC, gc.data(), sizeof(double) * 18 * N);
    std::memcpy(gradT, gt.data(), sizeof(double) * N);
    if (samples_out) std::memcpy(samples_out, rec.data(), nrec * sizeof(double));
    return SVSDF_OK;
}

}  // extern "C"
