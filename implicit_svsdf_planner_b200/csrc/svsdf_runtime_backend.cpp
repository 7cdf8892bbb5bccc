// svsdf_runtime_backend.cpp — the back-end optimisers: the host L-BFGS (svsdf_lbfgs_minimize, svsdf_optimize and its LMBM
// plug-in, svsdf_optimize_batch), the lock-step back end (svsdf_optimize_lockstep) and the device back end (svsdf_optimize_device).
#include <algorithm>
#include <chrono>
#include <cmath>

#include "host/lockstep.hpp"
#include "svsdf_runtime.h"

extern "C" {

void svsdf_default_lbfgs_params(svsdf_lbfgs_params *p) {
    host::LbfgsParams d;
    p->mem_size = d.mem_size; p->past = d.past; p->delta = d.delta; p->g_epsilon = d.g_epsilon;
    p->max_iterations = d.max_iterations; p->max_linesearch = d.max_linesearch; p->min_step = d.min_step;
    p->max_step = d.max_step; p->f_dec_coeff = d.f_dec_coeff; p->s_curv_coeff = d.s_curv_coeff;
    p->cautious_factor = d.cautious_factor; p->machine_prec = d.machine_prec;
    p->nonsmooth_restarts = 8;  // the SVSDF cost is non-smooth: restart across kinks, end with status 3 at a kink (svsdf.h)
}

static host::LbfgsParams to_host_params(const svsdf_lbfgs_params *params) {
    svsdf_lbfgs_params dp;
    svsdf_default_lbfgs_params(&dp);
    if (!params) params = &dp;
    host::LbfgsParams hp;
    hp.mem_size = params->mem_size; hp.past = params->past; hp.delta = params->delta; hp.g_epsilon = params->g_epsilon;
    hp.max_iterations = params->max_iterations; hp.max_linesearch = params->max_linesearch;
    hp.min_step = params->min_step; hp.max_step = params->max_step; hp.f_dec_coeff = params->f_dec_coeff;
    hp.s_curv_coeff = params->s_curv_coeff; hp.cautious_factor = params->cautious_factor;
    hp.machine_prec = params->machine_prec;
    hp.nonsmooth_restarts = params->nonsmooth_restarts;
    return hp;
}

// svsdf_optimize's return for a solver status: 0 is remapped to 1 (back_end_optimizer.cpp:66-69)
static int optimize_status(int solver_status) { return solver_status == 0 ? 1 : solver_status; }

// The checks of svsdf_optimize_lockstep and svsdf_optimize_device (`who`): the built-in L-BFGS only, and svsdf_optimize's checks of
// every problem with valid query points.
static int check_lockstep_problems(svsdf_ctx *ctx, const char *who, const svsdf_lockstep_problem *problems, int n) {
    if (ctx->lmbm) {
        ctx->err = std::string(who) + ": runs the built-in L-BFGS only; this context has an LMBM library set";
        return SVSDF_ERR_INVALID;
    }
    if (n < 0 || (n > 0 && !problems)) {
        ctx->err = std::string(who) + ": needs n >= 0 and the problem array";
        return SVSDF_ERR_INVALID;
    }
    for (int k = 0; k < n; ++k) {
        const svsdf_lockstep_problem &p = problems[k];
        if (!p.initS || !p.finalS || !p.opt_x || p.N < 2 || p.N > kMaxPieces || p.P < 0 || p.P > 2000000000LL || p.stride < 2 ||
            (p.P > 0 && !p.points)) {
            ctx->err = std::string(who) + ": problem " + std::to_string(k) +
                       ": needs initS, finalS, opt_x, 2 <= N <= 64, P >= 0, stride >= 2 and points when P > 0";
            return SVSDF_ERR_INVALID;
        }
    }
    return SVSDF_OK;
}

int svsdf_lbfgs_minimize(svsdf_eval_t eval, void *instance, double *x, int n, const svsdf_lbfgs_params *params,
                         svsdf_progress_t progress, void *user, svsdf_opt_stats *stats) {
    if (!eval || !x || n <= 0) return host::LBFGSERR_INVALID_N;
    host::Lbfgs solver(to_host_params(params));
    auto t0 = std::chrono::steady_clock::now();
    host::LbfgsResult R = solver.minimize(x, n, eval, instance, progress, user);
    auto t1 = std::chrono::steady_clock::now();
    fill_stats(stats, R.f, R.iterations, R.evaluations, R.status, std::chrono::duration<double>(t1 - t0).count(), 0.0);
    return R.status;
}

int svsdf_optimize(svsdf_ctx *ctx, const double *initS, const double *finalS, double *opt_x, int N,
                   const svsdf_lbfgs_params *params, svsdf_progress_t progress, void *user, double *T_out,
                   double *coeffs_out, svsdf_opt_stats *stats) {
    if (!ctx || !opt_x) return SVSDF_ERR_INVALID;
    int rc = svsdf_set_boundary(ctx, initS, finalS, N);
    if (rc) return rc;
    host::LbfgsParams hp = to_host_params(params);
    const int n = N + 3 * (N - 1);
    ctx->gpu_ms_total = 0.0;
    ctx->time_kernels = true;
    auto t0 = std::chrono::steady_clock::now();
    host::LbfgsResult R;
    if (ctx->lmbm) {  // the reference's own LMBM drives the callback (back_end_optimizer.cpp:29-36); this context's private instance
        struct Count { svsdf_ctx *ctx; int evals; svsdf_progress_t progress; void *user; int iters; } cnt{ctx, 0, progress, user, 0};
        double fx = 0.0;
        R.status = ctx->lmbm->optimize(
            n, opt_x, &fx,
            [](void *u, const double *xx, double *gg, const int nn) { Count *c = static_cast<Count *>(u); ++c->evals; return svsdf_evaluate(c->ctx, xx, gg, nn); }, &cnt,
            [](void *u, const double *xx, const int k) { Count *c = static_cast<Count *>(u); c->iters = k; return c->progress ? c->progress(c->user, xx, k) : 0; },
            &ctx->lmbm_params);
        R.f = fx;
        R.evaluations = cnt.evals;
        R.iterations = cnt.iters;
    } else {
        host::Lbfgs solver(hp);
        R = solver.minimize(opt_x, n, svsdf_evaluate, ctx, progress, user);
    }
    auto t1 = std::chrono::steady_clock::now();
    ctx->time_kernels = false;
    ctx->he.finish(opt_x, R, std::chrono::duration<double>(t1 - t0).count(), ctx->gpu_ms_total * 1e-3, T_out, coeffs_out, stats);
    // an evaluation that failed (points not set, CUDA error, duration >= 300 s) is an error of the run, whatever the
    // solver made of the NaN it was handed
    if (ctx->last_status != SVSDF_OK) return ctx->last_status;
    return optimize_status(R.status);
}

int svsdf_optimize_batch(svsdf_ctx *const *ctxs, int n_ctx, const svsdf_problem *problems, int n_problems, int N,
                         const svsdf_lbfgs_params *params, svsdf_next_problem_t next, void *next_user,
                         svsdf_opt_stats *stats_out, int *status_out, int64_t *points_out) {
    if (!problems && n_problems > 0) return SVSDF_ERR_INVALID;
    return run_pool(ctxs, n_ctx, n_problems, next, next_user, [&](svsdf_ctx *ctx, int k) -> int {
        const svsdf_problem &pr = problems[k];
        if (!pr.initS || !pr.finalS || !pr.opt_x) return SVSDF_ERR_INVALID;
        int rc;
        int64_t np = 0;
        if (pr.points) {
            rc = svsdf_set_points(ctx, pr.points, pr.P, pr.stride);
            np = pr.P;
        } else {
            rc = svsdf_extract_points(ctx, pr.waypoints_xy, pr.W, pr.half, pr.keepout_xy, pr.n_keepout, pr.clearance, &np);
        }
        if (rc != SVSDF_OK) {
            if (status_out) status_out[k] = rc;
            return rc;
        }
        if (points_out) points_out[k] = np;
        svsdf_opt_stats st;
        std::memset(&st, 0, sizeof(st));
        const int ret = svsdf_optimize(ctx, pr.initS, pr.finalS, pr.opt_x, N, params, nullptr, nullptr, pr.T_out, pr.coeffs_out, &st);
        if (stats_out) stats_out[k] = st;
        if (status_out) status_out[k] = ret;
        // solver codes (incl. negative line-search codes) are per-problem results; API / CUDA errors abort the call's status
        return (ret <= SVSDF_ERR_INVALID && ret > -1000) ? ret : SVSDF_OK;
    });
}

namespace {
// One slot of svsdf_optimize_lockstep: the host evaluation state of the problem in it and its device record.
struct LockstepSlot {
    HostEval he;
    MultiItem item;
    std::vector<double> out, pose_out;
    double *f0_out = nullptr;
    int last_status = SVSDF_OK;
    int evals = 0;
    double gpu_ms = 0.0;
    std::chrono::steady_clock::time_point t0;
};
}  // namespace

int svsdf_optimize_lockstep(svsdf_ctx *ctx, const svsdf_lockstep_problem *problems, int n, const svsdf_lbfgs_params *params, int max_in_flight,
                            svsdf_opt_stats *stats_out, int *status_out) {
    if (!ctx) return SVSDF_ERR_INVALID;
    if (const int rc = check_lockstep_problems(ctx, "svsdf_optimize_lockstep", problems, n)) return rc;
    if (const int rc = pose_ready(ctx, "svsdf_optimize_lockstep")) return rc;
    ctx->backend.lockstep_rounds = 0;
    ctx->backend.round_eval_ms = ctx->backend.round_backend_ms = 0.0;
    if (n == 0) return SVSDF_OK;
    CK(cudaSetDevice(ctx->device));
    const host::LbfgsParams hp = to_host_params(params);
    const int M = std::min(n, max_in_flight > 0 ? max_in_flight : 1024);
    if (M > kMaxMultiProblems) {
        ctx->err = "svsdf_optimize_lockstep: max_in_flight above 65535";
        return SVSDF_ERR_INVALID;
    }
    std::vector<LockstepSlot> slots(M);
    std::vector<MultiItem> items;
    int round_err = SVSDF_OK;
    auto enter = [&](int slot, int k) {
        LockstepSlot &s = slots[slot];
        const svsdf_lockstep_problem &p = problems[k];
        const int N = p.N;
        s.t0 = std::chrono::steady_clock::now();
        s.he.setup(p.initS, p.finalS, N);
        s.out.assign((size_t)19 * N + 2, 0.0);
        s.item = MultiItem();
        s.item.N = N; s.item.pts = p.points; s.item.P = p.P; s.item.stride = p.stride; s.item.out = s.out.data();
        if (ctx->pose_on) {
            s.pose_out.assign((size_t)4 * N * (ctx->pose.res + 1), 0.0);
            s.item.pose_out = s.pose_out.data();
        }
        s.f0_out = p.f0_out;
        s.last_status = SVSDF_OK;
        s.evals = 0;
        s.gpu_ms = 0.0;
        return host::LockstepEntry{p.opt_x, N + 3 * (N - 1), hp};
    };
    // the round: every slot's host forward half, one multi evaluation of all their trajectories and points, every slot's backward half
    auto round = [&](std::vector<host::LockstepEval> &evals) {
        const int count = (int)evals.size();
        items.resize(count);
#pragma omp parallel for schedule(dynamic)
        for (int j = 0; j < count; ++j) {
            LockstepSlot &s = slots[evals[j].slot];
            s.he.forward(evals[j].x);
            items[j] = s.item;
            items[j].T = s.he.times.data();
            items[j].coeffs = s.he.minco.getCoeffs();
        }
        float ms = 0.0f;
        const int rc = run_multi(ctx, items.data(), count, &ms);
        ctx->backend.round_eval_ms += ms;
        if (rc != SVSDF_OK && round_err == SVSDF_OK) round_err = rc;
#pragma omp parallel for schedule(dynamic)
        for (int j = 0; j < count; ++j) {
            host::LockstepEval &e = evals[j];
            LockstepSlot &s = slots[e.slot];
            s.gpu_ms += ms;
            // a failed evaluation hands the machine NaN, and its error stays the problem's status unless a later one succeeds
            s.last_status = rc != SVSDF_OK ? rc : items[j].rc;
            if (s.last_status != SVSDF_OK) {
                e.f = NAN;
                continue;
            }
            double pos = 0.0, other = 0.0;
            e.f = s.he.backward(s.out.data(), e.x, ctx->rho, ctx->pose_penalty(), s.pose_out.data(), ctx->dynamics(), e.g, &pos, &other);
            if (s.evals++ == 0 && s.f0_out) *s.f0_out = e.f;
        }
    };
    auto leave = [&](int slot, int k, const host::LbfgsResult &R) {
        LockstepSlot &s = slots[slot];
        const svsdf_lockstep_problem &p = problems[k];
        const double seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - s.t0).count();
        s.he.finish(p.opt_x, R, seconds, s.gpu_ms * 1e-3, p.T_out, p.coeffs_out, stats_out ? &stats_out[k] : nullptr);
        if (status_out) status_out[k] = s.last_status != SVSDF_OK ? s.last_status : optimize_status(R.status);
    };
    ctx->backend.lockstep_rounds = host::lockstep_run(n, M, enter, round, leave);
    return round_err;
}

int svsdf_optimize_device(svsdf_ctx *ctx, const svsdf_lockstep_problem *problems, int n, const svsdf_lbfgs_params *params, int max_in_flight,
                          svsdf_opt_stats *stats_out, int *status_out, int64_t *rounds_out) {
    if (!ctx) return SVSDF_ERR_INVALID;
    if (const int rc = check_lockstep_problems(ctx, "svsdf_optimize_device", problems, n)) return rc;
    if (max_in_flight > kMaxMultiProblems) {
        ctx->err = "svsdf_optimize_device: max_in_flight above 65535";
        return SVSDF_ERR_INVALID;
    }
    int Nmax = 2;
    for (int k = 0; k < n; ++k) Nmax = std::max(Nmax, problems[k].N);
    if (const int rc = pose_ready(ctx, "svsdf_optimize_device")) return rc;
    ctx->backend.lockstep_rounds = 0;
    ctx->backend.round_eval_ms = ctx->backend.round_backend_ms = 0.0;
    if (rounds_out) *rounds_out = 0;
    if (n == 0) return SVSDF_OK;
    CK(cudaSetDevice(ctx->device));
    const auto t0 = std::chrono::steady_clock::now();
    const host::LbfgsParams hp = to_host_params(params);
    if (const int bad = host::lbfgs_check(hp, 1)) {
        // parameters the solver refuses: every problem ends at once with the check's code, as svsdf_optimize ends (no evaluation; T
        // and the coefficients of the start point), and nothing is sized or launched
        for (int k = 0; k < n; ++k) {
            const svsdf_lockstep_problem &p = problems[k];
            HostEval he;
            he.setup(p.initS, p.finalS, p.N);
            host::LbfgsResult R;
            R.status = bad;
            he.finish(p.opt_x, R, 0.0, 0.0, p.T_out, p.coeffs_out, stats_out ? &stats_out[k] : nullptr);
            if (status_out) status_out[k] = bad;
        }
        return SVSDF_OK;
    }
    const int M = std::min(n, max_in_flight > 0 ? max_in_flight : 1024);
    const int64_t slot_doubles = backend_slot_doubles(hp, Nmax);
    // the call's problems, their result block (x0 in, then x, T, coeffs) and their resident points
    std::vector<BackendProblem> bp(n);
    std::vector<int64_t> pt_off(n);
    int64_t res_tot = 0, pts_tot = 0;
    for (int k = 0; k < n; ++k) {
        const svsdf_lockstep_problem &p = problems[k];
        std::memset(&bp[k], 0, sizeof(BackendProblem));
        bp[k].N = p.N;
        bp[k].res_off = res_tot;
        std::memcpy(bp[k].initS, p.initS, sizeof(bp[k].initS));
        std::memcpy(bp[k].finalS, p.finalS, sizeof(bp[k].finalS));
        res_tot += (4 * p.N - 3) + 19 * p.N;
        pt_off[k] = pts_tot;
        pts_tot += p.P;
    }
    if (pts_tot > INT32_MAX) {  // the resident points of the call share one index space (the multi kernels' int point index)
        ctx->err = "svsdf_optimize_device: more than 2^31 - 1 query points in one call";
        return SVSDF_ERR_INVALID;
    }
    CK(ctx->backend.d_slots.reserve(M));
    CK(ctx->backend.d_mem.reserve((size_t)M * slot_doubles));
    CK(ctx->backend.d_status.reserve(M));
    CK(ctx->backend.h_status.reserve(M));
    CK(ctx->backend.d_prob.reserve(n));
    CK(ctx->backend.d_result.reserve(n));
    CK(ctx->backend.d_res.reserve(res_tot));
    CK(ctx->backend.d_pts.reserve((size_t)2 * pts_tot));
    {
        std::vector<double> res(res_tot, 0.0);
        for (int k = 0; k < n; ++k) std::memcpy(res.data() + bp[k].res_off, problems[k].opt_x, sizeof(double) * (4 * bp[k].N - 3));
        CK(cudaMemcpyAsync(ctx->backend.d_prob, bp.data(), n * sizeof(BackendProblem), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(ctx->backend.d_res, res.data(), res_tot * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    }
    BackendArgs B;
    std::memset(&B, 0, sizeof(B));
    B.P = hp;
    B.rho = ctx->rho;
    B.dyn_on = ctx->dyn_on ? 1 : 0;
    B.dyn = ctx->dyn;
    B.pose_on = ctx->pose_on ? 1 : 0;
    B.pose = ctx->pose;
    B.Nmax = Nmax;
    B.slot_doubles = slot_doubles;
    B.slots = ctx->backend.d_slots;
    B.mem = ctx->backend.d_mem;
    B.status = ctx->backend.d_status;
    B.prob = ctx->backend.d_prob;
    B.result = ctx->backend.d_result;
    B.res = ctx->backend.d_res;
    std::vector<int> in_slot(M, -1), round_probs, entered;
    std::vector<double> seconds(n, 0.0), gpu_ms(n, 0.0);
    std::vector<char> finished(n, 0);
    std::vector<int64_t> round_valid_slots;
    int next = 0, round_err = SVSDF_OK;
    int64_t rounds = 0;
    bool timed = false, timed_init = false;
    // a CUDA error ends the call with that error in status_out of every problem not finished; the other outputs are then not written
    auto fail = [&](int rc) {
        if (status_out)
            for (int k = 0; k < n; ++k)
                if (!finished[k]) status_out[k] = rc;
        ctx->backend.lockstep_rounds = rounds;
        if (rounds_out) *rounds_out = rounds;
        return rc;
    };
#define CKB(call)                                                                       \
    do {                                                                                \
        cudaError_t e__ = (call);                                                       \
        if (e__ != cudaSuccess) {                                                       \
            ctx->err = std::string(#call) + ": " + cudaGetErrorString(e__);             \
            return fail(SVSDF_ERR_CUDA);                                                \
        }                                                                               \
    } while (0)
    // the round stage: [problems entering slots (pairs) | round items | problem table and CTA maps], each region rewritten only after
    // the stream synchronise that follows its last copy
    const size_t o_items = align16((size_t)2 * M * sizeof(int)), o_head0 = align16(o_items + (size_t)M * sizeof(BackendRoundItem));
    CKB(ctx->backend.h_round.reserve(o_head0));
    CKB(ctx->backend.d_round.reserve(o_head0));
    for (;;) {
        // problems enter the free slots: their points go up once, the machine starts and asks for its first evaluation
        int entering = 0;
        entered.clear();
        int *enter = reinterpret_cast<int *>(ctx->backend.h_round.get());
        for (int s = 0; s < M && next < n; ++s) {
            if (in_slot[s] >= 0) continue;
            const svsdf_lockstep_problem &p = problems[next];
            if (p.P > 0) {
                double *dst = ctx->backend.d_pts + 2 * pt_off[next];
                if (p.stride == 2) {
                    CKB(cudaMemcpyAsync(dst, p.points, (size_t)p.P * 16, cudaMemcpyHostToDevice, ctx->stream));
                } else {
                    std::vector<double> xy((size_t)2 * p.P);
                    pack_xy(xy.data(), p.points, p.P, p.stride);
                    CKB(cudaMemcpyAsync(dst, xy.data(), (size_t)p.P * 16, cudaMemcpyHostToDevice, ctx->stream));
                    CKB(cudaStreamSynchronize(ctx->stream));  // xy is about to go
                }
            }
            in_slot[s] = next;
            entered.push_back(next);
            enter[2 * entering] = s;
            enter[2 * entering + 1] = next;
            ++entering;
            ++next;
        }
        if (entering) {
            int *d_enter = reinterpret_cast<int *>(ctx->backend.d_round.get());
            CKB(cudaMemcpyAsync(d_enter, enter, (size_t)2 * entering * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
            CKB(cudaEventRecord(ctx->evk[2], ctx->stream));
            CKB(launch_backend_init(B, d_enter, entering, ctx->stream));
            CKB(cudaEventRecord(ctx->evk[3], ctx->stream));
            ctx->launches += 1;
            timed_init = true;
        }
        // 1. one small download: every slot's status
        CKB(cudaMemcpyAsync(ctx->backend.h_status, ctx->backend.d_status, (size_t)M * sizeof(BackendStatus), cudaMemcpyDeviceToHost, ctx->stream));
        CKB(cudaStreamSynchronize(ctx->stream));
        const BackendStatus *st = ctx->backend.h_status;
        const double now = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        if (timed_init) {  // the entering problems' first forward half
            float a = 0.0f;
            CKB(cudaEventElapsedTime(&a, ctx->evk[2], ctx->evk[3]));
            ctx->backend.round_backend_ms += a;
            for (int k : entered) gpu_ms[k] += a;
            timed_init = false;
        }
        if (timed) {  // the previous round's device time
            float a = 0.0f, b = 0.0f, c = 0.0f;
            CKB(cudaEventElapsedTime(&a, ctx->ev0, ctx->evk[0]));
            CKB(cudaEventElapsedTime(&b, ctx->evk[0], ctx->evk[1]));
            CKB(cudaEventElapsedTime(&c, ctx->evk[1], ctx->ev1));
            ctx->backend.round_eval_ms += b;
            ctx->backend.round_backend_ms += a + c;
            for (int k : round_probs) gpu_ms[k] += a + b + c;
            int64_t inside = 0;
            for (int64_t s : round_valid_slots) inside += st[s].n_inside;
            if (!round_valid_slots.empty()) ctx->multi_last_inside = inside;
            timed = false;
        }
        bool freed = false;
        for (int s = 0; s < M; ++s)
            if (in_slot[s] >= 0 && st[s].ask == host::LBFGS_DONE) {
                seconds[in_slot[s]] = now;
                finished[in_slot[s]] = 1;
                in_slot[s] = -1;
                freed = true;
            }
        if (freed && next < n) continue;
        // 2. the round: every slot asking for an evaluation, planned as run_multi plans (each problem keeps its single call's grid)
        MultiPlan pl;
        std::vector<BackendRoundItem> items;
        std::vector<PoseProblem> pp;  // the pose penalty's problems (pose on): every valid item's blob and records
        int64_t blob_tot = 0, pose_tot = 0;
        round_probs.clear();
        round_valid_slots.clear();
        for (int s = 0; s < M; ++s) {
            if (in_slot[s] < 0 || st[s].ask != host::LBFGS_EVAL) continue;
            const int k = in_slot[s];
            BackendRoundItem it;
            it.slot = s;
            it.rc = st[s].valid ? SVSDF_OK : SVSDF_ERR_INVALID;
            it.out_off = 0;
            it.blob_off = 0;
            it.pose_off = 0;
            round_probs.push_back(k);
            if (it.rc == SVSDF_OK) {
                const BlobLayout L = blob_layout(st[s].N, st[s].K1);
                MultiProblem m;
                std::memset(&m, 0, sizeof(m));
                m.blob_off = blob_tot;
                m.pt_off = pt_off[k];
                m.P = problems[k].P;
                m.blob_doubles = L.total;
                m.N = st[s].N;
                m.K1 = L.K1;
                it.blob_off = blob_tot;
                blob_tot += L.total;
                if (ctx->pose_on) {
                    it.pose_off = pose_tot;
                    pp.push_back(PoseProblem{it.blob_off, pose_tot});
                    pose_tot += (int64_t)m.N * (ctx->pose.res + 1);
                }
                pl.pr.push_back(m);
                round_valid_slots.push_back(s);
            }
            items.push_back(it);
        }
        const int count = (int)items.size();
        if (count == 0) break;  // nothing in flight and nothing left
        ++rounds;
        int rc = pl.pr.empty() ? SVSDF_OK : plan_multi(ctx, pl);
        if (rc == SVSDF_ERR_CUDA) return fail(rc);
        if (rc != SVSDF_OK) {  // the round fails: its error goes to every problem in it
            for (BackendRoundItem &it : items) it.rc = rc;
            if (round_err == SVSDF_OK) round_err = rc;
            pl = MultiPlan();
            pp.clear();
            round_valid_slots.clear();
        } else {
            for (int j = 0, v = 0; j < count; ++j)
                if (items[j].rc == SVSDF_OK) items[j].out_off = pl.pr[v++].out_off;
        }
        // 3. one small upload: the round items, the problem table and the CTA maps, the pose problems (the stage's earlier copies have
        // completed)
        const size_t o_pose = o_head0 + pl.head_bytes, bytes = o_pose + pp.size() * sizeof(PoseProblem);
        CKB(ctx->backend.h_round.reserve(bytes));
        CKB(ctx->backend.d_round.reserve(bytes));
        std::memcpy(ctx->backend.h_round + o_items, items.data(), (size_t)count * sizeof(BackendRoundItem));
        if (!pl.pr.empty()) pack_plan(pl, ctx->backend.h_round + o_head0);
        if (!pp.empty()) std::memcpy(ctx->backend.h_round + o_pose, pp.data(), pp.size() * sizeof(PoseProblem));
        CKB(cudaMemcpyAsync(ctx->backend.d_round + o_items, ctx->backend.h_round + o_items, bytes - o_items, cudaMemcpyHostToDevice, ctx->stream));
        const BackendRoundItem *d_items = reinterpret_cast<const BackendRoundItem *>(ctx->backend.d_round + o_items);
        // 4. the launches: blobs, the evaluation, the records into the machines
        CKB(cudaEventRecord(ctx->ev0, ctx->stream));
        if (!pl.pr.empty()) {
            CKB(ctx->backend.d_blobs.reserve(blob_tot));
            CKB(launch_backend_blob(B, d_items, count, ctx->backend.d_blobs, ctx->stream));
            ctx->launches += 1;
        }
        if (!pp.empty()) {  // the pose penalty's records, read by k_backend_backward
            CKB(ctx->d_pose_rec.reserve((size_t)4 * pose_tot));
            B.pose_rec = ctx->d_pose_rec;
            int max_N = 1;
            for (const MultiProblem &m : pl.pr) max_N = std::max(max_N, m.N);
            rc = launch_pose(ctx, ctx->pose, ctx->pose_half, ctx->backend.d_blobs, reinterpret_cast<const PoseProblem *>(ctx->backend.d_round + o_pose),
                             (int)pp.size(), max_N, ctx->d_pose_rec);
            if (rc) return fail(rc);
        }
        CKB(cudaEventRecord(ctx->evk[0], ctx->stream));
        double *records = nullptr;
        if (!pl.pr.empty()) {
            rc = launch_plan(ctx, pl, ctx->backend.d_round + o_head0, ctx->backend.d_blobs, ctx->backend.d_pts, nullptr, &records);
            if (rc) return fail(rc);
        }
        CKB(cudaEventRecord(ctx->evk[1], ctx->stream));
        CKB(launch_backend_backward(B, d_items, count, records, ctx->stream));
        ctx->launches += 1;
        CKB(cudaEventRecord(ctx->ev1, ctx->stream));
        timed = true;
    }
#undef CKB
    // the results: one download
    std::vector<BackendResult> R(n);
    std::vector<double> res(res_tot);
    CK(cudaMemcpyAsync(R.data(), ctx->backend.d_result, n * sizeof(BackendResult), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(res.data(), ctx->backend.d_res, res_tot * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (int k = 0; k < n; ++k) {
        const svsdf_lockstep_problem &p = problems[k];
        const int N = p.N, nv = 4 * N - 3;
        const double *x = res.data() + bp[k].res_off;
        std::memcpy(p.opt_x, x, sizeof(double) * nv);
        if (p.T_out) std::memcpy(p.T_out, x + nv, sizeof(double) * N);
        if (p.coeffs_out) std::memcpy(p.coeffs_out, x + nv + N, sizeof(double) * 18 * N);
        if (p.f0_out && R[k].f0_set) *p.f0_out = R[k].f0;
        fill_stats(stats_out ? &stats_out[k] : nullptr, R[k].f, R[k].iterations, R[k].evaluations, R[k].solver_status, seconds[k],
                   gpu_ms[k] * 1e-3);
        if (status_out) status_out[k] = R[k].status;
    }
    ctx->backend.lockstep_rounds = rounds;
    if (rounds_out) *rounds_out = rounds;
    return round_err;
}

int svsdf_round_times(const svsdf_ctx *ctx, double *eval_ms, double *backend_ms) {
    if (!ctx) return SVSDF_ERR_INVALID;
    if (eval_ms) *eval_ms = ctx->backend.round_eval_ms;
    if (backend_ms) *backend_ms = ctx->backend.round_backend_ms;
    return SVSDF_OK;
}

int svsdf_lockstep_rounds(const svsdf_ctx *ctx, int64_t *rounds) {
    if (!ctx || !rounds) return SVSDF_ERR_INVALID;
    *rounds = ctx->backend.lockstep_rounds;
    return SVSDF_OK;
}

int svsdf_set_lmbm_library(svsdf_ctx *ctx, const char *path, const svsdf_lmbm_params *params) {
    if (!ctx) return SVSDF_ERR_INVALID;
    if (ctx->lmbm) { svsdf_lmbm_close(ctx->lmbm); ctx->lmbm = nullptr; }
    if (!path) return SVSDF_OK;
    if (params) ctx->lmbm_params = *params; else svsdf_lmbm_default_params(&ctx->lmbm_params);
    const int rc = svsdf_lmbm_open(path, 1, &ctx->lmbm);
    if (rc) ctx->err = svsdf_lmbm_last_error();
    return rc;
}

}  // extern "C"
