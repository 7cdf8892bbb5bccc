// svsdf_runtime_front.cpp — the A* front end (K5): its shape kernels, the configuration-space map, node expansion, and whole
// searches on the host (svsdf_front_astar) or on the device (svsdf_front_astar_device).  Kernels: svsdf_frontend.cu.
#include <algorithm>
#include <cmath>

#include "host/astar.hpp"
#include "svsdf_runtime.h"

extern "C" {

int svsdf_front_init(svsdf_ctx *ctx, int kernel_size, int kernel_yaw_num, double occupancy_resolution, double front_end_safeh) {
    if (!ctx) return SVSDF_ERR_INVALID;
    if (kernel_size < 1 || kernel_size > kMaxKernelSize || (kernel_size % 2) == 0 || kernel_yaw_num < 1 || kernel_yaw_num > kMaxYawKernels ||
        !(occupancy_resolution > 0.0)) {
        ctx->err = "svsdf_front_init: kernel_size must be odd and <= 32, 1 <= kernel_yaw_num <= 64, resolution > 0";
        return SVSDF_ERR_INVALID;
    }
    if (ctx->shape.id == SH_POLYGON || ctx->shape.id == SH_MESH) {
        ctx->err = "svsdf_front_init: the reference defines no rotated kernels for the Polygon / mesh functors (Shape.hpp:1477 vs :267)";
        return SVSDF_ERR_INVALID;
    }
    CK(cudaSetDevice(ctx->device));
    ctx->front.ready = false;
    FrontParams F{};
    F.kernel_size = kernel_size;
    F.kernel_count = kernel_yaw_num;
    F.res = occupancy_resolution;
    F.safemargin = std::max(front_end_safeh, occupancy_resolution / 2);  // Shape.hpp:399
    const double PI = 3.14159265358979323846;                             // Shape.hpp:31
    const double yaw_res = 2 * PI / kernel_yaw_num;
    ctx->front.yaw.assign(kernel_yaw_num, 0.0);
    int ind = 0;
    for (double yaw = -PI; yaw < PI && ind < kernel_yaw_num; yaw += yaw_res, ind++) ctx->front.yaw[ind] = yaw;  // :401
    const int K = kernel_yaw_num, ks = kernel_size, bpr = (ks + 7) / 8;
    DeviceBuffer<double> d_yaw;
    DeviceBuffer<unsigned char> d_cells;
    CK(d_yaw.reserve(K));
    CK(d_cells.reserve((size_t)K * ks * ks));
    ctx->front.cells.assign((size_t)K * ks * ks, 0);
    CK(cudaMemcpyAsync(d_yaw, ctx->front.yaw.data(), K * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    CK(launch_front_cells(ctx->shape, F, d_yaw, d_cells, ctx->stream));
    CK(cudaMemcpyAsync(ctx->front.cells.data(), d_cells, ctx->front.cells.size(), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->launches += 1;
    // generateByteKernel (Shape.hpp:194-216) + the same rows as 32-bit masks (bit 31 - b <-> column b)
    static const unsigned char or_mask[8] = {0x80, 0x40, 0x20, 0x10, 0x08, 0x04, 0x02, 0x01};
    ctx->front.bytes.assign((size_t)K * ks * bpr, 0);
    std::vector<unsigned> rowmask((size_t)K * ks, 0u);
    for (int k = 0; k < K; ++k)
        for (int a = 0; a < ks; ++a)
            for (int b = 0; b < ks; ++b)
                if (ctx->front.cells[((size_t)k * ks + a) * ks + b]) {
                    ctx->front.bytes[((size_t)k * ks + a) * bpr + b / 8] |= or_mask[b % 8];
                    rowmask[(size_t)k * ks + a] |= 0x80000000u >> b;
                }
    CK(ctx->front.d_bytes.reserve(ctx->front.bytes.size()));
    CK(ctx->front.d_rowmask.reserve(rowmask.size()));
    CK(cudaMemcpy(ctx->front.d_bytes, ctx->front.bytes.data(), ctx->front.bytes.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(ctx->front.d_rowmask, rowmask.data(), rowmask.size() * sizeof(unsigned), cudaMemcpyHostToDevice));
    ctx->front.params = F;
    ctx->front.ready = true;
    return SVSDF_OK;
}

int svsdf_front_get_kernels(svsdf_ctx *ctx, double *yaw_out, unsigned char *cells_out, unsigned char *bytes_out) {
    if (!ctx) return SVSDF_ERR_INVALID;
    if (!ctx->front.ready) { ctx->err = "svsdf_front_get_kernels: call svsdf_front_init first"; return SVSDF_ERR_NOT_READY; }
    if (yaw_out) std::memcpy(yaw_out, ctx->front.yaw.data(), ctx->front.yaw.size() * sizeof(double));
    if (cells_out) std::memcpy(cells_out, ctx->front.cells.data(), ctx->front.cells.size());
    if (bytes_out) std::memcpy(bytes_out, ctx->front.bytes.data(), ctx->front.bytes.size());
    return SVSDF_OK;
}

static int front_params_with_map(svsdf_ctx *ctx, FrontParams &F, const char *who) {
    if (!ctx->front.ready) { ctx->err = std::string(who) + ": call svsdf_front_init first"; return SVSDF_ERR_NOT_READY; }
    if (!ctx->map()) { ctx->err = std::string(who) + ": map not set (svsdf_set_map)"; return SVSDF_ERR_NOT_READY; }
    F = ctx->front.params;
    F.X = ctx->map_X; F.Y = ctx->map_Y; F.h = ctx->map_h; F.row_bytes = ctx->map_row_bytes;
    F.out_words = (ctx->map_Y + 31) / 32;
    F.ox = ctx->map_ox; F.oy = ctx->map_oy; F.map_res = ctx->map_res;
    if (F.h != (F.kernel_size - 1) / 2) {
        ctx->err = std::string(who) + ": the map was packed for another kernel_size (its inflation must be (kernel_size - 1) / 2)";
        return SVSDF_ERR_INVALID;
    }
    if (F.res != F.map_res) {  // the reference has ONE conf.occupancy_resolution for the map and the shape kernels
        ctx->err = std::string(who) + ": svsdf_front_init's occupancy_resolution differs from the map resolution";
        return SVSDF_ERR_INVALID;
    }
    return SVSDF_OK;
}

// The node test's swept sub-volume: its half box and the kt lattice between a node and its child (sw_manager.hpp:1190)
static SubSwParams sub_sw_params(const FrontParams &F) {
    SubSwParams P{};
    P.half_box = (double)(F.kernel_size / 2 + 1);
    for (double kt = 0.0; kt <= 1.0 && P.nkt < 64; kt += 0.02) P.kt[P.nkt++] = kt;  // sw_manager.hpp:1190
    return P;
}

// SVSDF_ERR_INVALID with msg when one of the n cell indices (i, j) lies outside the map
static int cells_in_map(svsdf_ctx *ctx, const FrontParams &F, int64_t n, const int32_t *ij, const char *msg) {
    for (int64_t i = 0; i < n; ++i)
        if (ij[2 * i] < 0 || ij[2 * i] >= F.X || ij[2 * i + 1] < 0 || ij[2 * i + 1] >= F.Y) {
            ctx->err = msg;
            return SVSDF_ERR_INVALID;
        }
    return SVSDF_OK;
}

int svsdf_front_cspace(svsdf_ctx *ctx, uint32_t *words_out, float *ms_out, const uint32_t **dev_words_out) {
    if (!ctx) return SVSDF_ERR_INVALID;
    FrontParams F;
    int rc = front_params_with_map(ctx, F, "svsdf_front_cspace");
    if (rc != SVSDF_OK) return rc;
    CK(cudaSetDevice(ctx->device));
    const size_t n = (size_t)F.kernel_count * F.X * F.out_words;
    CK(ctx->front.d_cspace.reserve(n));
    CK(cudaEventRecord(ctx->ev0, ctx->stream));
    CK(launch_front_cspace(F, ctx->map(), ctx->front.d_rowmask, ctx->front.d_cspace, ctx->stream));
    CK(cudaEventRecord(ctx->ev1, ctx->stream));
    ctx->launches += 1;
    if (words_out) CK(cudaMemcpyAsync(words_out, ctx->front.d_cspace, n * sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (ms_out) CK(cudaEventElapsedTime(ms_out, ctx->ev0, ctx->ev1));
    if (dev_words_out) *dev_words_out = ctx->front.d_cspace;
    return SVSDF_OK;
}

int svsdf_front_expand(svsdf_ctx *ctx, int64_t n, const int32_t *node_ij, const double *node_yaw, unsigned char *ok_out, double *child_yaw_out,
                       unsigned char *parts_out) {
    if (!ctx || n < 0 || (n > 0 && (!node_ij || !node_yaw || !ok_out || !child_yaw_out))) return SVSDF_ERR_INVALID;
    FrontParams F;
    int rc = front_params_with_map(ctx, F, "svsdf_front_expand");
    if (rc != SVSDF_OK) return rc;
    if (n == 0) return SVSDF_OK;
    rc = cells_in_map(ctx, F, n, node_ij, "svsdf_front_expand: node index outside the map");
    if (rc != SVSDF_OK) return rc;
    const SubSwParams P = sub_sw_params(F);
    CK(cudaSetDevice(ctx->device));
    // One device scratch block and a pinned mirror of it: outputs first (child yaws [9n] f64 | ok [9n] | parts [9n], padded to
    // 8 bytes), then inputs (father yaws [n] f64 | node indices [2n] i32) — one copy in, one launch, one copy out.
    const size_t un = (size_t)n;
    const size_t out_bytes = (9 * un * 8 + 18 * un + 7) & ~(size_t)7, in_bytes = un * 8 + 2 * un * 4;
    CK(ctx->front.d_scratch.reserve(out_bytes + in_bytes + 64));
    CK(ctx->h_stage.reserve(out_bytes + in_bytes + 64));
    unsigned char *hb = ctx->h_stage, *db = ctx->front.d_scratch;
    double *d_cy = reinterpret_cast<double *>(db);
    unsigned char *d_ok = db + 9 * un * 8, *d_parts = d_ok + 9 * un;
    double *d_fy = reinterpret_cast<double *>(db + out_bytes);
    int *d_ij = reinterpret_cast<int *>(db + out_bytes + un * 8);
    std::memcpy(hb + out_bytes, node_yaw, un * 8);
    std::memcpy(hb + out_bytes + un * 8, node_ij, 2 * un * 4);
    cudaError_t e = cudaMemcpyAsync(db + out_bytes, hb + out_bytes, in_bytes, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = launch_front_expand(ctx->shape, F, P, ctx->map(), ctx->front.d_bytes, n, d_ij, d_fy, d_ok, d_cy, d_parts, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(hb, db, out_bytes, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e == cudaSuccess) {
        std::memcpy(child_yaw_out, hb, 9 * un * 8);
        std::memcpy(ok_out, hb + 9 * un * 8, 9 * un);
        if (parts_out) std::memcpy(parts_out, hb + 9 * un * 8 + 9 * un, 9 * un);
    }
    if (e != cudaSuccess) { ctx->err = std::string("svsdf_front_expand: ") + cudaGetErrorString(e); return SVSDF_ERR_CUDA; }
    ctx->launches += 1;
    return SVSDF_OK;
}

int svsdf_front_astar(svsdf_ctx *ctx, int n, const double *start_xy, const double *goal_xy, int max_path, double *paths_out, int32_t *len_out,
                      int32_t *expansions_out, int64_t *rounds_out) {
    if (!ctx || n < 0 || max_path < 1 || (n > 0 && (!start_xy || !goal_xy || !paths_out || !len_out))) return SVSDF_ERR_INVALID;
    FrontParams F;
    int rc = front_params_with_map(ctx, F, "svsdf_front_astar");
    if (rc != SVSDF_OK) return rc;
    host::AstarGrid G;
    G.X = F.X; G.Y = F.Y; G.ox = F.ox; G.oy = F.oy; G.res = F.map_res;
    host::AstarStats stats;
    auto expand = [&](int m, const int32_t *ij, const double *yaw, unsigned char *ok, double *cyaw) {
        return svsdf_front_expand(ctx, m, ij, yaw, ok, cyaw, nullptr);
    };
    rc = host::astar_batch(G, n, start_xy, goal_xy, max_path, paths_out, len_out, expansions_out, (int64_t)1 << 40, expand, &stats);
    if (rounds_out) *rounds_out = stats.rounds;
    return rc;
}

int svsdf_front_astar_device(svsdf_ctx *ctx, int n, const double *start_xy, const double *goal_xy, int max_path, int64_t max_expansions,
                             double *paths_out, int32_t *len_out, int32_t *expansions_out, int32_t *status_out, float *ms_out) {
    if (!ctx) return SVSDF_ERR_INVALID;
    if (n < 0 || max_path < 1 || max_expansions < 1 || (n > 0 && (!start_xy || !goal_xy || !paths_out || !len_out))) {
        ctx->err = "svsdf_front_astar_device: needs n >= 0, max_path >= 1, max_expansions >= 1 and the start, goal, path and length arrays";
        return SVSDF_ERR_INVALID;
    }
    FrontParams F;
    int rc = front_params_with_map(ctx, F, "svsdf_front_astar_device");
    if (rc != SVSDF_OK) return rc;
    if (ms_out) *ms_out = 0.0f;
    if (n == 0) return SVSDF_OK;
    CK(cudaSetDevice(ctx->device));
    // start / goal cells exactly as astar_batch finds them (isInMap, getGridIndex); -1: the search does not run
    const size_t un = (size_t)n;
    std::vector<int32_t> cells(4 * un);
    const double xmax = F.ox + F.X * F.map_res, ymax = F.oy + F.Y * F.map_res;
    auto in_map = [&](const double *v) { return !(v[0] < F.ox || v[1] < F.oy || v[0] > xmax || v[1] > ymax); };
    for (size_t q = 0; q < un; ++q) {
        const double *s = start_xy + 2 * q, *g = goal_xy + 2 * q;
        int32_t *c = &cells[4 * q];
        if (!in_map(s) || !in_map(g)) { c[0] = c[1] = c[2] = c[3] = -1; continue; }
        c[0] = host::astar_grid_index(s[0], F.ox, F.map_res, F.X); c[1] = host::astar_grid_index(s[1], F.oy, F.map_res, F.Y);
        c[2] = host::astar_grid_index(g[0], F.ox, F.map_res, F.X); c[3] = host::astar_grid_index(g[1], F.oy, F.map_res, F.Y);
    }
    const SubSwParams P = sub_sw_params(F);
    // Grid: min(n, resident CTAs, pool slots).  One slot per CTA: heap 16 B + g / f / yaw 24 B + father 4 B + id 1 B per entry, NS + 1
    // entries, rounded to 16 bytes; the pool is grow-only and capped at kAstarPoolCap (2 GiB: 8 slots of a 2400 x 2400 map).
    const int64_t NS = (int64_t)F.X * F.Y;
    const int64_t slot_bytes = ((NS + 1) * 45 + 15) & ~(int64_t)15;
    const int64_t kAstarPoolCap = (int64_t)2 << 30;
    const int64_t fit = kAstarPoolCap / slot_bytes;
    if (fit < 1) {
        ctx->err = "svsdf_front_astar_device: the map is too large for one search slot of the 2 GiB pool";
        return SVSDF_ERR_INVALID;
    }
    AstarArgs A{};
    int per_sm = 0;
    CK(launch_front_astar(ctx->shape, F, P, ctx->map(), ctx->front.d_bytes, A, 0, &per_sm, ctx->stream));
    int64_t grid = ctx->hooks.force_grid_astar > 0 ? ctx->hooks.force_grid_astar : std::min<int64_t>(n, (int64_t)std::max(per_sm, 1) * ctx->sm_count);
    grid = std::min(grid, fit);
    CK(ctx->front.d_astar_pool.reserve_exact((size_t)(grid * slot_bytes)));
    // One device block: cells [4n] i32 | len, expansions, status [3n] i32 | counter (padded to 16 bytes) | paths [n][max_path][3] f64.
    // Only the lengths come back first, then at most the longest returned path of every row.
    const size_t cells_bytes = 16 * un, out_bytes = 12 * un, head = (cells_bytes + out_bytes + 16 + 15) & ~(size_t)15;
    const size_t row = (size_t)max_path * 3 * sizeof(double);
    CK(ctx->front.d_scratch.reserve(head + un * row));
    CK(ctx->h_stage.reserve(cells_bytes + out_bytes));
    unsigned char *db = ctx->front.d_scratch;
    int32_t *hb = reinterpret_cast<int32_t *>(ctx->h_stage.get());
    std::memcpy(hb, cells.data(), cells_bytes);
    A.n = n; A.max_path = max_path; A.max_expansions = max_expansions;
    A.cells = reinterpret_cast<const int *>(db);
    A.len = reinterpret_cast<int *>(db + cells_bytes);
    A.expansions = A.len + un;
    A.status = A.len + 2 * un;
    A.next = reinterpret_cast<int *>(db + cells_bytes + out_bytes);
    A.paths = reinterpret_cast<double *>(db + head);
    A.pool = ctx->front.d_astar_pool;
    A.slot_bytes = slot_bytes;
    cudaError_t e = cudaMemcpyAsync(db, hb, cells_bytes, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(A.next, 0, sizeof(int), ctx->stream);
    if (e == cudaSuccess) e = cudaEventRecord(ctx->ev0, ctx->stream);
    if (e == cudaSuccess) e = launch_front_astar(ctx->shape, F, P, ctx->map(), ctx->front.d_bytes, A, (int)grid, nullptr, ctx->stream);
    if (e == cudaSuccess) e = cudaEventRecord(ctx->ev1, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(hb, A.len, out_bytes, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { ctx->err = std::string("svsdf_front_astar_device: ") + cudaGetErrorString(e); return SVSDF_ERR_CUDA; }
    ctx->launches += 1;
    int32_t lmax = 0;
    for (size_t q = 0; q < un; ++q) lmax = std::max(lmax, hb[q]);
    std::memcpy(len_out, hb, un * 4);
    if (expansions_out) std::memcpy(expansions_out, hb + un, un * 4);
    if (status_out) std::memcpy(status_out, hb + 2 * un, un * 4);
    if (lmax > 0) CK(cudaMemcpy2DAsync(paths_out, row, A.paths, row, (size_t)lmax * 3 * sizeof(double), un, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (ms_out) CK(cudaEventElapsedTime(ms_out, ctx->ev0, ctx->ev1));
    return SVSDF_OK;
}

int svsdf_front_check_kernel_value(svsdf_ctx *ctx, int64_t n, const double *father_yaw, const int32_t *ind_xy, unsigned char *ok_out,
                                   double *child_yaw_out) {
    if (!ctx || n < 0 || (n > 0 && (!father_yaw || !ind_xy || !ok_out || !child_yaw_out))) return SVSDF_ERR_INVALID;
    FrontParams F;
    int rc = front_params_with_map(ctx, F, "svsdf_front_check_kernel_value");
    if (rc != SVSDF_OK) return rc;
    if (n == 0) return SVSDF_OK;
    rc = cells_in_map(ctx, F, n, ind_xy, "svsdf_front_check_kernel_value: cell index outside the map");
    if (rc != SVSDF_OK) return rc;
    CK(cudaSetDevice(ctx->device));
    const size_t un = (size_t)n;
    CK(ctx->front.d_scratch.reserve(un * 8 + un * 8 + 2 * un * 4 + un + 64));
    double *d_fy = reinterpret_cast<double *>(ctx->front.d_scratch.get());
    double *d_cy = d_fy + un;
    int *d_ind = reinterpret_cast<int *>(d_cy + un);
    unsigned char *d_ok = reinterpret_cast<unsigned char *>(d_ind + 2 * un);
    cudaError_t e = cudaMemcpyAsync(d_fy, father_yaw, n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_ind, ind_xy, 2 * n * sizeof(int), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = launch_front_check(F, ctx->map(), ctx->front.d_bytes, n, d_fy, d_ind, d_ok, d_cy, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ok_out, d_ok, n, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(child_yaw_out, d_cy, n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { ctx->err = std::string("svsdf_front_check_kernel_value: ") + cudaGetErrorString(e); return SVSDF_ERR_CUDA; }
    ctx->launches += 1;
    return SVSDF_OK;
}

}  // extern "C"
