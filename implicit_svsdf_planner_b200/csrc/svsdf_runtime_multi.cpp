// svsdf_runtime_multi.cpp — n problems per set of launches: the multi-problem launch plan (also run by the device back end),
// svsdf_cost_grad_multi, and svsdf_cost_grad_batch's pool of contexts.
#include <algorithm>
#include <cmath>

#include "svsdf_runtime.h"

int plan_multi(svsdf_ctx *ctx, MultiPlan &pl) {
    for (size_t j = 0; j < pl.pr.size(); ++j) {
        MultiProblem &m = pl.pr[j];
        Occupancy occ;
        int rc = occupancy(ctx, m.N, m.blob_doubles, &occ);
        if (rc) return rc;
        const OuterPlan plan = outer_plan(ctx, m.P, occ);
        const int G = plan.grid, batched = plan.batched;
        m.flag_off = pl.flag_tot; m.part_off = pl.part_tot; m.out_off = pl.out_tot; m.grid = G;
        std::vector<int> &mp = batched ? pl.map_b : pl.map_s;
        for (int v = 0; v < G; ++v) { mp.push_back((int)j); mp.push_back(v); }
        pl.pt_round += m.P;
        pl.pt_span = std::max(pl.pt_span, m.pt_off + m.P);
        pl.flag_tot += (m.P + 15) & ~(int64_t)15;
        pl.part_tot += (int64_t)G * (19 * m.N + 1);
        pl.out_tot += 19 * m.N + 2;
        pl.max_K1 = std::max(pl.max_K1, m.K1);
        pl.max_N = std::max(pl.max_N, m.N);
        pl.max_blob = std::max(pl.max_blob, m.blob_doubles);
        pl.smax_blob[batched] = std::max(pl.smax_blob[batched], m.blob_doubles);
        pl.smax_N[batched] = std::max(pl.smax_N[batched], m.N);
        if (batched) pl.max_rounds = std::max(pl.max_rounds, outer_rounds(m.P, G));
    }
    for (int b = 0; b < 2; ++b)
        if (outer_smem_doubles(pl.smax_blob[b], pl.smax_N[b], 1) * sizeof(double) > kMaxDynSmemBytes) {
            ctx->err = "svsdf: trajectory blob does not fit in shared memory";
            return SVSDF_ERR_INVALID;
        }
    if (!pl.map_b.empty()) {
        Occupancy occ;
        int rc = occupancy(ctx, pl.smax_N[1], pl.smax_blob[1], &occ);
        if (rc) return rc;
        pl.chunk = outer_chunk(ctx, occ, pl.max_rounds, pl.smax_blob[1], pl.smax_N[1]);
    }
    pl.o_ms = align16(pl.pr.size() * sizeof(MultiProblem));
    pl.o_mb = align16(pl.o_ms + pl.map_s.size() * sizeof(int));
    pl.head_bytes = align16(pl.o_mb + pl.map_b.size() * sizeof(int));
    return SVSDF_OK;
}

void pack_plan(const MultiPlan &pl, unsigned char *h) {
    std::memcpy(h, pl.pr.data(), pl.pr.size() * sizeof(MultiProblem));
    if (!pl.map_s.empty()) std::memcpy(h + pl.o_ms, pl.map_s.data(), pl.map_s.size() * sizeof(int));
    if (!pl.map_b.empty()) std::memcpy(h + pl.o_mb, pl.map_b.data(), pl.map_b.size() * sizeof(int));
}

int launch_plan(svsdf_ctx *ctx, const MultiPlan &pl, const unsigned char *d, double *d_blobs, const double *d_points, const PointQuery *pq,
                double **records) {
    const int m = (int)pl.pr.size();
    const int64_t pt_span = pl.pt_span, pt_round = pl.pt_round;
    // scratch: flags | inside t* | inside lists | contributions | pieces | partials | out | tot | counts | slot offsets
    const size_t s_flag = 0, s_ts = align16(s_flag + (size_t)pl.flag_tot + 16), s_list = align16(s_ts + (size_t)pt_span * 8),
                 s_con = align16(s_list + (size_t)pt_span * 4), s_pc = align16(s_con + (size_t)pt_round * 160),
                 s_part = align16(s_pc + (size_t)pt_round * 4), s_out = align16(s_part + (size_t)pl.part_tot * 8),
                 s_tot = align16(s_out + (size_t)pl.out_tot * 8), s_cnt = align16(s_tot + (size_t)pl.out_tot * 8), s_off = align16(s_cnt + (size_t)m * 4),
                 s_bytes = align16(s_off + (size_t)(m + 1) * 4);
    CK(ctx->multi.d_scratch.reserve(s_bytes));
    if ((size_t)m + 1 > ctx->multi.d_tickets.capacity()) {  // a new block: its tickets start at zero
        CK(ctx->multi.d_tickets.reserve(m + 1));
        CK(cudaMemsetAsync(ctx->multi.d_tickets, 0, ctx->multi.d_tickets.capacity() * sizeof(unsigned int), ctx->stream));
    }
    unsigned char *sc = ctx->multi.d_scratch;
    KernelArgs A;
    std::memset(&A, 0, sizeof(A));
    A.blob = d_blobs;
    A.points_xy = d_points;
    A.cp = ctx->cp;
    A.partials = reinterpret_cast<double *>(sc + s_part);
    A.want_reduce = pq ? 0 : 1;
    if (pq) { A.out_sdf = pq->sdf; A.out_tstar = pq->tstar; }
    const bool outer_only = pq && pq->outer_only;
    A.want_gsip = outer_only ? 0 : 1;
    A.inside_flag = sc + s_flag;
    A.inside_tstar = reinterpret_cast<double *>(sc + s_ts);
    A.inside_list = reinterpret_cast<int *>(sc + s_list);
    A.gsip_contrib = reinterpret_cast<double *>(sc + s_con);
    A.gsip_piece = reinterpret_cast<int *>(sc + s_pc);
    A.eval_counter = ctx->count_evals ? ctx->d_eval_counter.get() : nullptr;
    MultiArgs M;
    std::memset(&M, 0, sizeof(M));
    M.n = m;
    M.prob = reinterpret_cast<const MultiProblem *>(d);
    M.ins_count = reinterpret_cast<int *>(sc + s_cnt);
    M.ins_off = reinterpret_cast<int *>(sc + s_off);
    M.compact_ticket = ctx->multi.d_tickets;
    M.tickets = ctx->multi.d_tickets + 1;
    M.out = reinterpret_cast<double *>(sc + s_out);
    M.tot = reinterpret_cast<double *>(sc + s_tot);
    const ScaleSched *Z = ctx->scaled ? &ctx->sched : nullptr;
    const Kernels &K = kernels(ctx);
    CK(K.pose_multi(d_blobs, M, pl.max_K1, ctx->stream));
    int launches = 1;
    for (int b = 0; b < 2; ++b) {
        const std::vector<int> &mp = b ? pl.map_b : pl.map_s;
        if (mp.empty()) continue;
        M.cta_map = reinterpret_cast<const int *>(d + (b ? pl.o_mb : pl.o_ms));
        A.outer_chunk = b ? pl.chunk : 1;
        CK(K.multi(b, A, M, ctx->shape, Z, (int)(mp.size() / 2),
                   outer_smem_doubles(pl.smax_blob[b], pl.smax_N[b], A.outer_chunk) * sizeof(double), 0, ctx->sm_count, ctx->stream));
        ++launches;
    }
    M.cta_map = nullptr;
    if (outer_only) {  // the per-point values are written; nothing else runs
        ctx->launches += launches;
        return SVSDF_OK;
    }
    CK(K.compact_multi(A.inside_flag, A.inside_list, M, ctx->stream));
    const GsipPlan gp = gsip_plan(ctx, pq ? -1 : ctx->multi_last_inside);  // the variant svsdf_query would pick
    CK(K.multi(2, A, M, ctx->shape, Z, gp.grid, (size_t)pl.max_blob * sizeof(double), gp.wide, ctx->sm_count, ctx->stream));
    launches += 2;
    if (!pq) {
        CK(K.finalize_multi(A.partials, A.gsip_contrib, A.gsip_piece, M, pl.max_N, ctx->stream));
        launches += 1;
    }
    ctx->launches += launches;
    if (records) *records = M.out;
    return SVSDF_OK;
}

int run_multi(svsdf_ctx *ctx, MultiItem *items, int n, float *ms, const PointQuery *pq) {
    if (ms) *ms = 0.0f;
    CK(cudaSetDevice(ctx->device));
    MultiPlan pl;
    std::vector<int> who;
    std::vector<BlobLayout> lay;
    std::vector<double> dur;
    int64_t blob_tot = 0, pt_tot = 0;
    for (int k = 0; k < n; ++k) {
        MultiItem &it = items[k];
        if (it.rc != SVSDF_OK) continue;
        BlobLayout L;
        double D = 0.0;
        const char *msg = nullptr;
        if (it.P < 0 || it.P > 2000000000LL || (!pq && (it.stride < 2 || (it.P > 0 && !it.pts) || !it.out)) ||
            traj_layout(it.N, it.T, it.coeffs, L, D, &msg) != SVSDF_OK) {
            it.rc = SVSDF_ERR_INVALID;
            continue;
        }
        MultiProblem m;
        std::memset(&m, 0, sizeof(m));
        m.blob_off = blob_tot; m.pt_off = pt_tot;
        m.P = it.P; m.blob_doubles = L.total; m.N = it.N; m.K1 = L.K1;
        pl.pr.push_back(m);
        who.push_back(k);
        lay.push_back(L);
        dur.push_back(D);
        blob_tot += L.total;
        pt_tot += it.P;
    }
    const int m = (int)pl.pr.size();
    if (m == 0) return SVSDF_OK;
    int rc = plan_multi(ctx, pl);
    if (rc) return rc;
    // the pose penalty's problems: the items that want its records
    std::vector<PoseProblem> pp;
    std::vector<int> pose_item;
    int64_t pose_tot = 0;
    if (!pq)
        for (int j = 0; j < m; ++j)
            if (items[who[j]].pose_out) {
                pp.push_back(PoseProblem{pl.pr[j].blob_off, pose_tot});
                pose_item.push_back(j);
                pose_tot += (int64_t)pl.pr[j].N * (ctx->pose.res + 1);
            }
    // packed inputs: problem table | CTA maps (sparse, batched) | blobs | points (x, y; not with pq) | pose problems
    const size_t o_blob = pl.head_bytes, o_pts = align16(o_blob + (size_t)blob_tot * 8),
                 o_pose = align16(o_pts + (pq ? 0 : (size_t)pt_tot * 16)), in_bytes = align16(o_pose + pp.size() * sizeof(PoseProblem));
    CK(ctx->multi.h_in.reserve(in_bytes));
    CK(ctx->multi.d_in.reserve(in_bytes));
    // the previous call's copy has completed (every call ends with a stream synchronise)
    unsigned char *h = ctx->multi.h_in, *d = ctx->multi.d_in;
    pack_plan(pl, h);
    for (int j = 0; j < m; ++j) {
        const MultiItem &it = items[who[j]];
        fill_blob(reinterpret_cast<double *>(h + o_blob) + pl.pr[j].blob_off, lay[j], it.T, it.coeffs, dur[j]);
        if (pq) continue;
        pack_xy(reinterpret_cast<double *>(h + o_pts) + 2 * pl.pr[j].pt_off, it.pts, it.P, it.stride);
    }
    if (!pp.empty()) std::memcpy(h + o_pose, pp.data(), pp.size() * sizeof(PoseProblem));
    CK(ctx->multi.h_out.reserve(pl.out_tot + 4 * pose_tot));
    CK(cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
    if (ms) CK(cudaEventRecord(ctx->ev0, ctx->stream));
    if (!pp.empty()) {
        CK(ctx->d_pose_rec.reserve((size_t)4 * pose_tot));
        rc = launch_pose(ctx, ctx->pose, ctx->pose_half, reinterpret_cast<const double *>(d + o_blob),
                         reinterpret_cast<const PoseProblem *>(d + o_pose), (int)pp.size(), pl.max_N, ctx->d_pose_rec);
        if (rc) return rc;
    }
    double *records = nullptr;
    rc = launch_plan(ctx, pl, d, reinterpret_cast<double *>(d + o_blob), pq ? pq->pts : reinterpret_cast<const double *>(d + o_pts), pq,
                     &records);
    if (rc) return rc;
    if (pq) return SVSDF_OK;
    if (ms) CK(cudaEventRecord(ctx->ev1, ctx->stream));
    CK(cudaMemcpyAsync(ctx->multi.h_out, records, (size_t)pl.out_tot * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (!pp.empty())
        CK(cudaMemcpyAsync(ctx->multi.h_out + pl.out_tot, ctx->d_pose_rec, (size_t)pose_tot * 32, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (ms) CK(cudaEventElapsedTime(ms, ctx->ev0, ctx->ev1));
    for (size_t q = 0; q < pp.size(); ++q) {
        const int j = pose_item[q];
        std::memcpy(items[who[j]].pose_out, ctx->multi.h_out + pl.out_tot + 4 * pp[q].rec_off,
                    (size_t)pl.pr[j].N * (ctx->pose.res + 1) * 32);
    }
    int64_t inside = 0;
    for (int j = 0; j < m; ++j) {
        const int nout = 19 * pl.pr[j].N + 2;
        const double *o = ctx->multi.h_out + pl.pr[j].out_off;
        std::memcpy(items[who[j]].out, o, (size_t)nout * sizeof(double));
        inside += (int64_t)o[nout - 1];
    }
    ctx->multi_last_inside = inside;
    return SVSDF_OK;
}

extern "C" {

int svsdf_cost_grad_multi(svsdf_ctx *ctx, int n, const svsdf_multi_problem *problems) {
    if (!ctx) return SVSDF_ERR_INVALID;
    if (n < 0 || n > kMaxMultiProblems || (n > 0 && !problems)) {
        ctx->err = "svsdf_cost_grad_multi: needs 0 <= n <= 65535 and the problem array";
        return SVSDF_ERR_INVALID;
    }
    std::vector<MultiItem> items(n);
    std::vector<std::vector<double>> outs(n);
    for (int k = 0; k < n; ++k) {
        const svsdf_multi_problem &p = problems[k];
        BlobLayout L;
        double D;
        const char *msg = "svsdf_cost_grad_multi: invalid points or null outputs";
        if (!p.cost_io || !p.gradT_io || !p.gradC_io || p.P < 0 || p.P > 2000000000LL || p.stride < 2 || (p.P > 0 && !p.points) ||
            traj_layout(p.N, p.T, p.coeffs, L, D, &msg) != SVSDF_OK) {
            ctx->err = std::string("problem ") + std::to_string(k) + ": " + msg;
            return SVSDF_ERR_INVALID;
        }
        outs[k].assign((size_t)19 * p.N + 2, 0.0);
        MultiItem &it = items[k];
        it.N = p.N; it.T = p.T; it.coeffs = p.coeffs; it.pts = p.points; it.P = p.P; it.stride = p.stride; it.out = outs[k].data();
    }
    if (n == 0) return SVSDF_OK;
    int rc = run_multi(ctx, items.data(), n, nullptr);
    if (rc) return rc;
    for (int k = 0; k < n; ++k)
        if (items[k].rc != SVSDF_OK) {  // cannot happen after the checks above; never hand back a record that was not computed
            ctx->err = std::string("svsdf_cost_grad_multi: problem ") + std::to_string(k) + " was refused";
            return items[k].rc;
        }
    bool finite = true;
    for (int k = 0; k < n; ++k) {
        const svsdf_multi_problem &p = problems[k];
        const double *o = outs[k].data();
        const int N = p.N;
        *p.cost_io += o[0];
        for (int e = 0; e < 18 * N; ++e) p.gradC_io[e] += o[1 + e];
        for (int i = 0; i < N; ++i) p.gradT_io[i] += o[1 + 18 * N + i];
        if (p.n_inside_out) *p.n_inside_out = (int64_t)o[1 + 19 * N];
        finite = finite && std::isfinite(o[0]);
    }
    return finite ? SVSDF_OK : SVSDF_ERR_NONFINITE;
}

int svsdf_cost_grad_batch(svsdf_ctx *const *ctxs, int n_ctx, int n_problems, int N, const double *const *pts, const int64_t *P,
                          int stride, const double *T, const double *coeffs, double *cost_io, double *gradT_io, double *gradC_io) {
    if (n_problems > 0 && (!pts || !P || !T || !coeffs || !cost_io || !gradT_io || !gradC_io)) return SVSDF_ERR_INVALID;
    return run_pool(ctxs, n_ctx, n_problems, nullptr, nullptr, [&](svsdf_ctx *ctx, int k) -> int {
        int rc = svsdf_set_points(ctx, pts[k], P[k], stride);
        if (rc != SVSDF_OK) return rc;
        return svsdf_cost_grad(ctx, N, T + (size_t)k * N, coeffs + (size_t)k * 18 * N, cost_io + k, gradT_io + (size_t)k * N,
                               gradC_io + (size_t)k * 18 * N);
    });
}

}  // extern "C"
