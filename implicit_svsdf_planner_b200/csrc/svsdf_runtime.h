// svsdf_runtime.h — what the units of the host runtime (svsdf_runtime_*.cpp) share; private to libsvsdf_b200.so.
//
// The runtime owns the device buffers (query points resident in HBM, trajectory blob, per-CTA partials, inside-point lists), the
// CUDA stream, pinned staging memory, the host MINCO spline and the host L-BFGS, and launches the sm_90a kernels of
// svsdf_kernels.cuh.  There is deliberately no CPU implementation of the hot path in this library: if CUDA is unavailable
// svsdf_create fails.  Every unit is compiled with -ffp-contract=off (build.py: RUNTIME_FLAGS), which keeps HostEval, MINCO and
// the winding-number builder bit-exact.
#pragma once

#include <cuda_runtime.h>

#include <atomic>
#include <cstring>
#include <map>
#include <string>
#include <thread>
#include <tuple>
#include <vector>

#include "../../include/svsdf.h"
#include "host/lbfgs.hpp"
#include "host/minco.hpp"
#include "svsdf_backend.h"
#include "svsdf_launch.h"
#include "svsdf_types.h"

using namespace svsdf;

// One run's svsdf_opt_stats (stats may be null), shared by both back ends and svsdf_lbfgs_minimize.
inline void fill_stats(svsdf_opt_stats *stats, double f, int iterations, int evaluations, int status, double seconds, double gpu_seconds) {
    if (!stats) return;
    stats->final_cost = f;
    stats->iterations = iterations;
    stats->evaluations = evaluations;
    stats->status = status;
    stats->seconds = seconds;
    stats->gpu_seconds = gpu_seconds;
}

// The host half of one back-end evaluation (back_end_optimizer.hpp:353-398), shared by svsdf_evaluate and the lock-step back end
// (svsdf_optimize_lockstep).  forward(): tau -> T and MINCO (coefficients, energy and its partial gradients), before the device
// evaluation; backward(): adds the device record, the pose penalty (pose not null) and the dynamics penalty (dyn not null), propagates
// through MINCO and adds rho * sum(T).
struct HostEval {
    host::MincoS3NU minco;
    int N = 0;
    std::vector<double> times, gradByTimes, partialGradByTimes, partialGradByCoeffs, gradByPoints, adj, dynPartial;
    double energy = 0.0;

    void setup(const double *initS, const double *finalS, int n_pieces) {
        N = n_pieces;
        minco.setConditions(initS, finalS, N);
        times.assign(N, 0.0);
        gradByTimes.assign(N, 0.0);
        partialGradByTimes.assign(N, 0.0);
        partialGradByCoeffs.assign((size_t)18 * N, 0.0);
        gradByPoints.assign((size_t)3 * (N - 1), 0.0);
        adj.assign((size_t)18 * N, 0.0);
        dynPartial.assign(N, 0.0);
    }
    host::BackendEvalView view() {
        return host::BackendEvalView{minco.view(),           times.data(),        gradByTimes.data(), partialGradByTimes.data(),
                                     partialGradByCoeffs.data(), gradByPoints.data(), adj.data(), dynPartial.data()};
    }
    void forward(const double *x) { energy = host::backend_forward(view(), x); }
    // o: the device record [cost, gradC (18N), gradT (N), n_inside] of the trajectory forward() built; pose_rec: its pose penalty's
    // sample records (read when pose is not null)
    double backward(const double *o, const double *x, double rho, const host::PoseParams *pose, const double *pose_rec,
                    const host::DynamicsParams *dyn, double *g, double *pos_out, double *other_out) {
        return host::backend_backward(view(), energy, o, x, rho, pose, pose_rec, dyn, g, pos_out, other_out);
    }
    // The final trajectory from the solver's returned iterate x (optimize_traj_lmbm does the same on success and failure,
    // back_end_optimizer.cpp:44-94) and the run's statistics.
    void finish(const double *x, const host::LbfgsResult &R, double seconds, double gpu_seconds, double *T_out, double *coeffs_out,
                svsdf_opt_stats *stats) {
        for (int i = 0; i < N; ++i) times[i] = host::forwardT(x[i]);
        minco.setParameters(x + N, times.data());
        if (T_out) std::memcpy(T_out, times.data(), sizeof(double) * N);
        if (coeffs_out) std::memcpy(coeffs_out, minco.getCoeffs(), sizeof(double) * 18 * N);
        fill_stats(stats, R.f, R.iterations, R.evaluations, R.status, seconds, gpu_seconds);
    }
};

// An owning block of device memory (or, PINNED, page-locked host memory) of T.  reserve(n) is grow-only and keeps no contents: when the
// block holds fewer than n elements it is freed and n + n / 2 + 4096 are allocated (reserve_exact: n).  A reserved buffer is never null,
// even for n = 0.
template <class T, bool PINNED = false>
class Buffer {
  public:
    Buffer() = default;
    Buffer(Buffer &&o) noexcept : p_(o.p_), cap_(o.cap_) { o.p_ = nullptr; o.cap_ = 0; }
    Buffer &operator=(Buffer &&o) noexcept {
        std::swap(p_, o.p_);
        std::swap(cap_, o.cap_);
        return *this;
    }
    ~Buffer() { release(); }
    cudaError_t reserve(size_t n) { return p_ && n <= cap_ ? cudaSuccess : allocate(n + n / 2 + 4096); }
    cudaError_t reserve_exact(size_t n) { return p_ && n <= cap_ ? cudaSuccess : allocate(n); }
    void release() {
        if (p_) PINNED ? cudaFreeHost(p_) : cudaFree(p_);
        p_ = nullptr;
        cap_ = 0;
    }
    size_t capacity() const { return cap_; }
    T *get() const { return p_; }
    operator T *() const { return p_; }

  private:
    cudaError_t allocate(size_t n) {
        release();
        void *q = nullptr;
        const cudaError_t e = PINNED ? cudaMallocHost(&q, n * sizeof(T)) : cudaMalloc(&q, n * sizeof(T));
        if (e != cudaSuccess) return e;
        p_ = static_cast<T *>(q);
        cap_ = n;
        return cudaSuccess;
    }
    T *p_ = nullptr;
    size_t cap_ = 0;
};
template <class T>
using DeviceBuffer = Buffer<T>;
template <class T>
using PinnedBuffer = Buffer<T, true>;

// (resident single-problem k_outer, k_gsip CTAs per SM) of one trajectory size; chunk: the most batches per descent pass (<=
// kOuterChunkMax) whose work area leaves k_outer's residency what it is with one
struct Occupancy {
    int outer, gsip, chunk;
};

// The reference's LMBM library as a plug-in (lmbm.h:214-221): one dlopen of (a private copy of) the file per handle.
struct svsdf_lmbm {
    void *dl = nullptr;
    // lmbm::lmbm_optimize(int, double*, double*, lmbm_evaluate_t, void*, lmbm_progress_t, lmbm_parameter_t*)
    int (*optimize)(int, double *, double *, svsdf_eval_t, void *, svsdf_progress_t, svsdf_lmbm_params *) = nullptr;
};

// The test hooks, read ONCE at svsdf_create from the environment (read_test_hooks); -1 = not set.
struct TestHooks {
    // SVSDF_FORCE_GRID_OUTER / SVSDF_FORCE_BATCHED: exercise the batched schedule on small inputs
    int force_grid_outer = -1;
    int force_batched = -1;
    // SVSDF_FORCE_GSIP_WIDE = 0 / 1: the 8-warp or the 22-warp k_gsip for queries and cost evaluations alike; SVSDF_FORCE_GRID_GSIP =
    // n > 0: k_gsip grid, 1 = one CTA walks every slot
    int force_gsip_wide = -1;
    int force_grid_gsip = -1;
    // SVSDF_FORCE_GRID_ASTAR = n > 0 sets k_astar_search's grid (1 = one CTA runs every search on the same slot)
    int force_grid_astar = -1;
    // SVSDF_FORCE_POSE_WINDOWS = 0 (none: every layer evaluates the trajectory), 1 (layer 2 only) or 2 (layers 2 and 3), whatever
    // pose_windows' rule says
    int force_pose_windows = -1;
    // SVSDF_FORCE_OUTER_CHUNK = n > 0 sets the batches per descent pass of the batched k_outer (outer_chunk), whatever the rounds and
    // the residency say; still clipped to kOuterChunkMax and the shared memory
    int force_outer_chunk = -1;
};

// One context.  What one unit alone reads and writes sits in a sub-struct named for it; the rest is shared.
struct svsdf_ctx {
    svsdf_config cfg;
    std::string shape_name;
    ShapeParams shape;
    CostParams cp;
    double rho = 3.8;
    int device = 0;
    bool strict = false;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaEvent_t evk[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};  // per-kernel timing marks
    bool mark_kernels = false;
    float last_kernel_ms[4] = {0, 0, 0, 0};  // pose table, k_outer, k_compact + k_gsip, k_finalize
    std::string err;
    int64_t launches = 0;
    TestHooks hooks;

    // query points
    // packed xy: the caller's block (svsdf_set_points_device) when one is set, else points_buf
    DeviceBuffer<double> points_buf;
    const double *points_ext = nullptr;
    const double *points() const { return points_ext ? points_ext : points_buf.get(); }
    int64_t P = 0;
    // scratch sized by P
    DeviceBuffer<unsigned char> d_flag;
    DeviceBuffer<double> d_inside_tstar;
    DeviceBuffer<int> d_inside_list;
    DeviceBuffer<double> d_gsip_contrib;
    DeviceBuffer<int> d_gsip_piece;
    DeviceBuffer<int> d_n_inside;
    DeviceBuffer<unsigned long long> d_eval_counter;
    bool count_evals = false;
    // trajectory blob
    DeviceBuffer<double> d_blob;
    PinnedBuffer<double> h_blob;
    BlobLayout layout{};
    int traj_N = 0;
    double traj_D = 0.0;
    std::map<std::tuple<int, int, int>, Occupancy> occ_cache;  // (N, blob doubles, scaled) -> resident CTAs per SM
    // deformable robot (svsdf_set_scale): the scaled kernels run with this schedule
    bool scaled = false;
    ScaleSched sched{};
    int64_t last_n_inside = -1;  // interior points seen by the previous cost evaluation (picks the k_gsip variant)
    int64_t multi_last_inside = -1;  // inside points of the previous multi evaluation (picks the k_gsip_multi variant)
    // pose windows of choiceTInit layers 2 and 3 (svsdf_types.h:PoseRec), rebuilt with the layer-1 table: [layer 2 | layer 3]
    DeviceBuffer<PoseRec> d_win;
    int win_layers = 0;  // 0: none built, 1: layer 2, 2: layers 2 and 3
    // reduction
    DeviceBuffer<double> d_partials;
    DeviceBuffer<double> d_out;  // 1 + 19N + 1
    DeviceBuffer<double> d_tot;  // 19N + 1 (finalize scratch)
    DeviceBuffer<unsigned int> d_ticket;
    PinnedBuffer<double> h_out;
    PinnedBuffer<unsigned char> h_stage;  // staging for results download and the small uploads of the other entry points

    // packed map kernel (K3), written by svsdf_runtime_map.cpp
    // the caller's block (svsdf_set_map_device) when one is set, else map_buf
    DeviceBuffer<unsigned char> map_buf;
    const unsigned char *map_ext = nullptr;
    const unsigned char *map() const { return map_ext ? map_ext : map_buf.get(); }
    int map_X = 0, map_Y = 0, map_h = 0, map_row_bytes = 0;
    int map_Z = 1;             // z layers held on the device (svsdf_set_map3d), each in the 2-D layout; layer 0 first
    double map_ox = 0, map_oy = 0, map_oz = 0, map_res = 0;
    bool map3d = false;

    // optimiser state (R3/R4)
    HostEval he;
    bool have_boundary = false;
    double cost_pos = 0, cost_other = 0, cost_total = 0;
    int n_evaluate = 0;
    double gpu_ms_total = 0.0;
    bool time_kernels = false;
    int last_status = 0;
    svsdf_lmbm *lmbm = nullptr;          // svsdf_set_lmbm_library: this context's private instance of the reference's LMBM
    svsdf_lmbm_params lmbm_params;
    // speed and yaw-rate limits (svsdf_set_dynamics): every back-end evaluation of this context adds their penalty when dyn_on
    bool dyn_on = false;
    host::DynamicsParams dyn{};
    const host::DynamicsParams *dynamics() const { return dyn_on ? &dyn : nullptr; }
    // the pose-sampled obstacle penalty (svsdf_set_pose_penalty): every back-end evaluation of this context adds it when pose_on; it
    // gathers its cells from the 3-D map (map3d: the map came from svsdf_set_map3d).  d_pose_rec: the sample records of a call
    bool pose_on = false;
    host::PoseParams pose{};
    double pose_half[3] = {0, 0, 0};
    const host::PoseParams *pose_penalty() const { return pose_on ? &pose : nullptr; }
    DeviceBuffer<double> d_pose_rec;

    // svsdf_runtime_context.cpp: the mesh functor's device arrays (SH_MESH), referenced by shape
    struct {
        DeviceBuffer<double> d_tri;  // kMeshStride doubles per face
        DeviceBuffer<unsigned int> d_fwn_child;  // the winding-number hierarchy (host/fwn_bvh.hpp)
        DeviceBuffer<float> d_fwn_data, d_fwn_cbox, d_fwn_trif;
    } mesh;
    // svsdf_runtime_context.cpp: svsdf_set_points has its own pinned stage and does NOT wait for its copies: the kernels that follow
    // are ordered behind them on the context's stream, and the host goes on (builds the trajectory blob) while the DMA runs.  ev marks
    // the end of the last upload: the next svsdf_set_points (which overwrites the stage) and svsdf_device_ptr_points (which hands the
    // buffer to other streams) wait on it.
    struct {
        PinnedBuffer<double> h_stage;
        cudaEvent_t ev = nullptr;
        bool inflight = false;
    } upload;
    // svsdf_runtime_eval.cpp: svsdf_query's per-point outputs
    struct {
        DeviceBuffer<double> d_points, d_sdf, d_ts, d_grad;
        DeviceBuffer<int> d_rounds;
    } query;
    // svsdf_runtime_front.cpp: the A* front end's collision kernels (K5), its device scratch and the search slots of
    // svsdf_front_astar_device (exactly sized, see kAstarPoolCap)
    struct {
        bool ready = false;
        FrontParams params{};
        std::vector<double> yaw;
        std::vector<unsigned char> cells, bytes;
        DeviceBuffer<unsigned char> d_bytes;
        DeviceBuffer<unsigned> d_rowmask;
        DeviceBuffer<unsigned> d_cspace;
        DeviceBuffer<unsigned char> d_scratch;
        DeviceBuffer<unsigned char> d_astar_pool;
    } front;
    // svsdf_runtime_map.cpp: svsdf_extract_points' per-CTA counts and per-layer totals
    struct {
        DeviceBuffer<int> d_block_counts;
        DeviceBuffer<int64_t> d_n_total;
    } extract;
    // svsdf_runtime_multi.cpp: packed inputs of a multi evaluation (one pinned stage mirrored by one device block, one copy in),
    // scratch, pinned outputs (one copy out)
    struct {
        PinnedBuffer<unsigned char> h_in;
        DeviceBuffer<unsigned char> d_in;
        DeviceBuffer<unsigned char> d_scratch;
        PinnedBuffer<double> h_out;
        DeviceBuffer<unsigned int> d_tickets;  // [0] k_compact_multi's, [1 + k] problem k's k_finalize_multi ticket; zero between calls
    } multi;
    // svsdf_runtime_backend.cpp: the last svsdf_optimize_lockstep / svsdf_optimize_device; svsdf_optimize_device's slots (machine
    // state, storage, status), the call's problems, results and resident points, the round's blobs
    struct {
        int64_t lockstep_rounds = 0;  // rounds
        double round_eval_ms = 0.0, round_backend_ms = 0.0;  // their device time: evaluation kernels, back-end kernels (svsdf_round_times)
        DeviceBuffer<BackendSlot> d_slots;
        DeviceBuffer<double> d_mem, d_res, d_pts, d_blobs;
        DeviceBuffer<BackendStatus> d_status;
        PinnedBuffer<BackendStatus> h_status;
        DeviceBuffer<BackendProblem> d_prob;
        DeviceBuffer<BackendResult> d_result;
        DeviceBuffer<unsigned char> d_round;
        PinnedBuffer<unsigned char> h_round;
    } backend;
    // svsdf_runtime_swept.cpp: svsdf_swept_contour's device buffers (per corner, per needed corner, per CTA, outputs);
    // svsdf_map_clearance's (header, samples and per-CTA counts; band bits per map word; band cells)
    struct {
        DeviceBuffer<unsigned char> d_corner, d_point, d_small, d_out;
        DeviceBuffer<unsigned char> d_cl_small, d_cl_band, d_cl_point;
    } swept;
};

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e__ = (call);                                                                  \
        if (e__ != cudaSuccess) {                                                                  \
            ctx->err = std::string(#call) + ": " + cudaGetErrorString(e__);                        \
            return SVSDF_ERR_CUDA;                                                                 \
        }                                                                                          \
    } while (0)

// The launchers of one kernel variant, kKernels[strict][scaled]: FMA contraction or not (-fmad=false, the reference's rounding), rigid
// or deformable robot.  The scaled variants share the rigid units' pose table, finalize, shape evaluation and multi-problem helpers.
struct Kernels {
    decltype(&fast::query_occupancy) query_occupancy;
    decltype(&fast::launch_cost_kernels) cost_kernels;
    decltype(&fast::launch_pose_table) pose_table;
    decltype(&fast::launch_finalize) finalize;
    decltype(&fast::launch_shape_eval) shape_eval;
    decltype(&fast::launch_sincos) sincos;
    decltype(&fast_multi::launch_multi) multi;
    decltype(&fast_multi::launch_pose_multi) pose_multi;
    decltype(&fast_multi::launch_compact_multi) compact_multi;
    decltype(&fast_multi::launch_finalize_multi) finalize_multi;
    decltype(&fast::launch_pose) pose;
};
extern const Kernels kKernels[2][2];
inline const Kernels &kernels(const svsdf_ctx *ctx) { return kKernels[ctx->strict][ctx->scaled]; }

inline size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }

// n rows of `stride` doubles (x and y first) packed into x, y pairs at dst
inline void pack_xy(double *dst, const double *src, int64_t n, int stride) {
    if (stride == 2) {
        if (n) std::memcpy(dst, src, (size_t)n * 2 * sizeof(double));
        return;
    }
    for (int64_t i = 0; i < n; ++i) {
        dst[2 * i] = src[i * stride];
        dst[2 * i + 1] = src[i * stride + 1];
    }
}

// ---- argument checks shared by a setter and another entry point (svsdf_runtime_context.cpp) ------------------------------------
bool scale_valid(const svsdf_scale &z);
bool dynamics_valid(const svsdf_dynamics &d);
host::DynamicsParams to_host_dynamics(const svsdf_dynamics &d);
int pose_penalty_check(svsdf_ctx *ctx, const svsdf_pose_penalty &p, const char *who);

// ---- single-problem evaluation (svsdf_runtime_eval.cpp) -------------------------------------------------------------------------
int ensure_scratch(svsdf_ctx *ctx, int64_t P);
// updateTraj's checks (sw_manager.hpp:376-385) and the blob layout of one trajectory; on failure the message is in *err
int traj_layout(int N, const double *T, const double *coeffs, BlobLayout &L, double &D, const char **err);
// the host part of the blob (everything before the pose rows, which k_pose_table fills)
void fill_blob(double *h, const BlobLayout &L, const double *T, const double *coeffs, double D);
// updateTraj (sw_manager.hpp:376-385) + the layer-1 lattice of choiceTInit (:538-581): builds the blob in pinned memory, uploads it
// and (launch_pose) launches the pose-table kernel for an evaluation of P points.
int upload_traj(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, int64_t P, bool launch_pose = true);
// Runs K1 (+compact, K2) (+finalize) on the uploaded trajectory.  Inputs resident on the device.
int run_kernels(svsdf_ctx *ctx, const double *d_points, int64_t P, bool reduce, bool gsip, double *o_sdf, double *o_ts, double *o_grad,
                int *o_rounds);
// With the pose penalty on (svsdf_set_pose_penalty) the context needs a 3-D map: checked before any launch.
int pose_ready(svsdf_ctx *ctx, const char *who);
// The pose penalty's sample records (4 doubles each) of n trajectories into rec: problem k's blob at blobs + prob[k].blob_off, its
// N (res + 1) records from record prob[k].rec_off (prob null: one problem, blob at blobs, records from 0).  max_N: the most pieces.
int launch_pose(svsdf_ctx *ctx, const host::PoseParams &pp, const double *half, const double *blobs, const PoseProblem *prob, int n,
                int max_N, double *rec);

// The launch-plan rule of k_outer and k_gsip, shared by the single call and every problem of a multi evaluation (which is what gives
// a multi problem the bits of its single call).
int occupancy(svsdf_ctx *ctx, int N, int blob, Occupancy *occ);
struct OuterPlan {
    int grid, batched;
};
OuterPlan outer_plan(const svsdf_ctx *ctx, int64_t P, const Occupancy &occ);
int outer_chunk(const svsdf_ctx *ctx, const Occupancy &occ, int64_t rounds, int blob, int N);
int64_t outer_rounds(int64_t P, int grid);
struct GsipPlan {
    int wide, grid;
};
GsipPlan gsip_plan(const svsdf_ctx *ctx, int64_t prev_inside);

// ---- n problems per set of launches (svsdf_runtime_multi.cpp) -------------------------------------------------------------------
struct MultiItem {
    int N = 0;
    const double *T = nullptr, *coeffs = nullptr;
    const double *pts = nullptr;  // P rows of `stride` doubles, x and y first
    int64_t P = 0;
    int stride = 2;
    double *out = nullptr;        // host record [cost, gradC (18N), gradT (N), n_inside]
    double *pose_out = nullptr;   // not null: also the pose penalty's N (res + 1) sample records (svsdf_optimize_lockstep, pose on)
    int rc = SVSDF_OK;
};

// svsdf_map_clearance_multi's and svsdf_swept_contour_multi's evaluation: the items' points already on the device (concatenated in
// item order; MultiItem::pts and ::out are not used) and svsdf_query's per-point values at the same places, instead of the cost and
// gradient (tstar may be null).  outer_only: svsdf_query(outer_only = 1)'s values, the outer solve alone (no k_compact_multi, no
// k_gsip_multi).
struct PointQuery {
    const double *pts;
    double *sdf, *tstar;
    bool outer_only = false;
};

// The planning and launch sequence of one multi evaluation, shared by run_multi and svsdf_optimize_device.  The caller fills each
// problem's blob_off, pt_off, P, blob_doubles, N and K1; plan_multi gives it the virtual grid and schedule of its single call (occupancy /
// outer_plan: what gives it the single call's bits), the CTA maps and the scratch offsets.
struct MultiPlan {
    std::vector<MultiProblem> pr;
    std::vector<int> map_s, map_b;
    int64_t flag_tot = 0, part_tot = 0, out_tot = 0;
    int64_t pt_round = 0;  // points of the round's problems (inside contributions)
    int64_t pt_span = 0;   // points the pt_off values span (inside t* and lists are indexed by pt_off)
    int max_K1 = 1, max_N = 1, max_blob = 2;
    int smax_blob[2] = {0, 0}, smax_N[2] = {1, 1};  // per k_outer_multi launch (sparse, batched): the shared memory is sized by its largest
    int64_t max_rounds = 1;  // most batches a warp of the batched launch owns
    int chunk = 1;           // the batched launch's batches per descent pass (outer_chunk at its largest blob and N)
    size_t o_ms = 0, o_mb = 0, head_bytes = 0;        // packed head: problem table | CTA maps (sparse, batched)
};
int plan_multi(svsdf_ctx *ctx, MultiPlan &pl);
void pack_plan(const MultiPlan &pl, unsigned char *h);
// The launches of a planned evaluation whose packed head is at d (device) and blobs at d_blobs: k_pose_table_multi, k_outer_multi per
// schedule that occurs, k_compact_multi and k_gsip_multi (not with pq->outer_only) and k_finalize_multi (not with pq).  *records: the per-problem records [cost,
// gradC (18N), gradT (N), n_inside] at out_off (device).
int launch_plan(svsdf_ctx *ctx, const MultiPlan &pl, const unsigned char *d, double *d_blobs, const double *d_points, const PointQuery *pq,
                double **records);
// One cost + gradient evaluation of every item with rc == SVSDF_OK, in one set of launches.  Items whose trajectory or points are
// invalid get rc = SVSDF_ERR_INVALID and take no part; a CUDA error fails the call (and every item).  *ms: device time of the launches.
// With pq: the per-point query of every item instead (no reduction, no finalize, nothing downloaded; multi_last_inside is kept).
int run_multi(svsdf_ctx *ctx, MultiItem *items, int n, float *ms, const PointQuery *pq = nullptr);

// ---- batch variants: a pool of contexts, one worker thread each, dynamic hand-out of problem indices ----------------------------
template <class Body>
int run_pool(svsdf_ctx *const *ctxs, int n_ctx, int n_problems, svsdf_next_problem_t next, void *next_user, Body body) {
    if (!ctxs || n_ctx < 1 || n_problems < 0) return SVSDF_ERR_INVALID;
    for (int c = 0; c < n_ctx; ++c)
        if (!ctxs[c]) return SVSDF_ERR_INVALID;
    std::atomic<int> counter{0};
    std::atomic<int> first_err{SVSDF_OK};
    auto worker = [&](int c) {
        for (;;) {
            const int k = next ? next(next_user) : counter.fetch_add(1);
            if (k < 0 || k >= n_problems) break;
            const int rc = body(ctxs[c], k);
            if (rc != SVSDF_OK) {
                int expected = SVSDF_OK;
                first_err.compare_exchange_strong(expected, rc);
            }
        }
    };
    if (n_ctx == 1) {
        worker(0);
    } else {
        std::vector<std::thread> th;
        th.reserve(n_ctx);
        for (int c = 0; c < n_ctx; ++c) th.emplace_back(worker, c);
        for (auto &t : th) t.join();
    }
    return first_err.load();
}
