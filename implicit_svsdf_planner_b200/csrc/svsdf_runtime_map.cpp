// svsdf_runtime_map.cpp — the occupancy map (svsdf_set_map[_device], svsdf_set_map3d) and the query points extracted from it
// (svsdf_extract_points[3d]).  Kernels: svsdf_extract.cu.
#include <algorithm>

#include "svsdf_runtime.h"

extern "C" {

static int set_map_meta(svsdf_ctx *ctx, int X, int Y, int kernel_size, double ox, double oy, double res) {
    if (X <= 0 || Y <= 0 || kernel_size < 1 || (kernel_size & 1) == 0 || !(res > 0.0)) {
        ctx->err = "svsdf_set_map: bad map geometry (kernel_size must be odd, res > 0)";
        return SVSDF_ERR_INVALID;
    }
    ctx->map_X = X; ctx->map_Y = Y; ctx->map_h = (kernel_size - 1) / 2;
    ctx->map_row_bytes = (Y + 2 * ctx->map_h + 7) / 8;
    ctx->map_ox = ox; ctx->map_oy = oy; ctx->map_oz = 0.0; ctx->map_res = res;
    ctx->map_Z = 1;
    ctx->map3d = false;
    return SVSDF_OK;
}

int svsdf_set_map(svsdf_ctx *ctx, const unsigned char *kernel_bytes, int X, int Y, int kernel_size, double origin_x,
                  double origin_y, double res) {
    if (!ctx || !kernel_bytes) return SVSDF_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    int rc = set_map_meta(ctx, X, Y, kernel_size, origin_x, origin_y, res);
    if (rc) return rc;
    const size_t bytes = (size_t)(X + 2 * ctx->map_h) * ctx->map_row_bytes;
    ctx->map_ext = nullptr;
    CK(ctx->map_buf.reserve(bytes));
    CK(cudaMemcpyAsync(ctx->map_buf, kernel_bytes, bytes, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return SVSDF_OK;
}

int svsdf_set_map_device(svsdf_ctx *ctx, const unsigned char *dev_kernel_bytes, int X, int Y, int kernel_size,
                         double origin_x, double origin_y, double res) {
    if (!ctx || !dev_kernel_bytes) return SVSDF_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    int rc = set_map_meta(ctx, X, Y, kernel_size, origin_x, origin_y, res);
    if (rc) return rc;
    ctx->map_buf.release();
    ctx->map_ext = dev_kernel_bytes;
    return SVSDF_OK;
}

// generateMapKernel's layout (PCSmap_manager.h:39-78: [(X + 2h)][(Y + 2h)][ceil((Z + 2h) / 8)] bytes, z bits MSB first) is re-packed on
// the host, once per map, into Z layers of the 2-D layout the kernels read ([(X + 2h)][ceil((Y + 2h) / 8)], y bits MSB first); layer 0 is
// what generateMapKernel2D would have produced, so the front-end kernels see the same map as with svsdf_set_map.
int svsdf_set_map3d(svsdf_ctx *ctx, const unsigned char *kernel_bytes, int X, int Y, int Z, int kernel_size, const double *origin_xyz,
                    double res) {
    if (!ctx || !kernel_bytes || !origin_xyz || Z < 1 || Z > kMaxMapLayers) return SVSDF_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    int rc = set_map_meta(ctx, X, Y, kernel_size, origin_xyz[0], origin_xyz[1], res);
    if (rc) return rc;
    const int h = ctx->map_h;
    const size_t layer = (size_t)(X + 2 * h) * ctx->map_row_bytes;
    const int zb = (Z + 2 * h + 7) / 8;
    std::vector<unsigned char> L(layer * (size_t)Z, 0);
    for (int x = 0; x < X; ++x)
        for (int y = 0; y < Y; ++y) {
            const unsigned char *col = kernel_bytes + ((size_t)(x + h) * (Y + 2 * h) + (size_t)(y + h)) * zb;
            for (int z = 0; z < Z; ++z) {
                const int fz = z + h;
                if (col[fz / 8] & (0x80u >> (fz % 8))) {
                    const int fy = y + h;
                    L[(size_t)z * layer + (size_t)(x + h) * ctx->map_row_bytes + fy / 8] |= (unsigned char)(0x80u >> (fy % 8));
                }
            }
        }
    const size_t bytes = L.size();
    ctx->map_ext = nullptr;
    CK(ctx->map_buf.reserve(bytes));
    CK(cudaMemcpyAsync(ctx->map_buf, L.data(), bytes, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->map_Z = Z;
    ctx->map_oz = origin_xyz[2];
    ctx->map3d = true;
    return SVSDF_OK;
}

// Shared by the flat and the 3-D entry points.  wp: W x 3 waypoint centres, half: box half sizes (x, y, z).
static int extract_impl(svsdf_ctx *ctx, const char *who, const double *wp, int W, const double *half, const double *keepout_xy,
                        int n_keepout, double clearance, int64_t *n_points) {
    if (!ctx->map()) { ctx->err = std::string(who) + ": map not set"; return SVSDF_ERR_NOT_READY; }
    CK(cudaSetDevice(ctx->device));
    ExtractArgs E;
    std::memset(&E, 0, sizeof(E));
    E.X = ctx->map_X; E.Y = ctx->map_Y; E.h = ctx->map_h; E.row_bytes = ctx->map_row_bytes;
    E.ox = ctx->map_ox; E.oy = ctx->map_oy; E.res = ctx->map_res;
    E.W = W;
    const int Z = ctx->map_Z;
    const double lo[3] = {E.ox, E.oy, ctx->map_oz};
    const double hi[3] = {E.ox + (double)E.X * E.res, E.oy + (double)E.Y * E.res, ctx->map_oz + (double)Z * E.res};  // boundary_xyzmax
    const int size[3] = {E.X, E.Y, Z};
    auto box = [&](const double *c, int idx[3][2]) { map_index_box(c, half, lo, hi, size, E.res, idx); };
    int bz1[kMaxWaypoints + 1], bz2[kMaxWaypoints + 1];  // slot 0: the box around tmp_pos, slot w + 1: waypoint w
    {
        const double tmp_pos[3] = {999.0, 999.0, 999.0};  // plan_manager.cpp:152
        int idx[3][2];
        box(tmp_pos, idx);
        E.px1 = idx[0][0]; E.px2 = idx[0][1]; E.py1 = idx[1][0]; E.py2 = idx[1][1];
        bz1[0] = idx[2][0]; bz2[0] = idx[2][1];
    }
    int rxmin = E.X, rxmax = -1, rymin = E.Y, rymax = -1;
    for (int w = 0; w < W; ++w) {
        int idx[3][2];
        box(wp + 3 * w, idx);
        E.bx1[w] = idx[0][0]; E.bx2[w] = idx[0][1]; E.by1[w] = idx[1][0]; E.by2[w] = idx[1][1];
        bz1[w + 1] = idx[2][0]; bz2[w + 1] = idx[2][1];
        rxmin = std::min(rxmin, E.bx1[w]); rxmax = std::max(rxmax, E.bx2[w]);
        rymin = std::min(rymin, E.by1[w]); rymax = std::max(rymax, E.by2[w]);
    }
    E.rx1 = rxmin;
    E.wy1 = (rymin + E.h) / 32;
    const int wy2 = (rymax + E.h) / 32;
    E.nW = wy2 - E.wy1 + 1;
    E.n_items = (long long)(rxmax - rxmin + 1) * E.nW;
    E.n_keepout = n_keepout;
    E.clearance = clearance;
    for (int q = 0; q < 2 * n_keepout; ++q) E.keepout[q] = keepout_xy[q];
    const int n_blocks = (int)((E.n_items + 255) / 256);
    const size_t need_counts = (size_t)(n_blocks + 1) * (size_t)Z;
    CK(ctx->extract.d_block_counts.reserve(need_counts));
    CK(ctx->extract.d_n_total.reserve(kMaxMapLayers));
    const size_t layer = (size_t)(E.X + 2 * E.h) * E.row_bytes;
    auto layer_args = [&](int k) {
        ExtractArgs Ek = E;
        Ek.map = ctx->map() + (size_t)k * layer;
        for (int w = 0; w < W; ++w) {
            Ek.act[w] = (k >= bz1[w + 1] && k <= bz2[w + 1]) ? 1 : 0;
            Ek.excl[w] = (k >= bz1[w] && k <= bz2[w]) ? 1 : 0;
        }
        return Ek;
    };
    for (int k = 0; k < Z; ++k) {
        CK(launch_extract_count(layer_args(k), ctx->extract.d_block_counts + (size_t)k * (n_blocks + 1), n_blocks, ctx->extract.d_n_total + k, ctx->stream));
        ctx->launches += 2;
    }
    int64_t totals[kMaxMapLayers];
    CK(cudaMemcpyAsync(totals, ctx->extract.d_n_total, (size_t)Z * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    int64_t total = 0;
    for (int k = 0; k < Z; ++k) total += totals[k];
    if (total > 2000000000LL) { ctx->err = std::string(who) + ": too many points"; return SVSDF_ERR_INVALID; }
    ctx->points_ext = nullptr;
    CK(ctx->points_buf.reserve((size_t)total * 2));
    int64_t base = 0;
    for (int k = 0; k < Z; ++k) {  // layer-major output: layer 0's cells in ascending (i * Y + j) order, then layer 1's, ...
        CK(launch_extract_write(layer_args(k), ctx->extract.d_block_counts + (size_t)k * (n_blocks + 1), n_blocks, ctx->points_buf + 2 * base, totals[k], ctx->stream));
        ctx->launches += 1;
        base += totals[k];
    }
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->P = total;
    ctx->last_n_inside = -1;
    if (n_points) *n_points = total;
    return ensure_scratch(ctx, total);
}

int svsdf_extract_points(svsdf_ctx *ctx, const double *waypoints_xy, int W, double half, const double *keepout_xy,
                         int n_keepout, double clearance, int64_t *n_points) {
    if (!ctx || !waypoints_xy || W < 1 || W > kMaxWaypoints || n_keepout < 0 || n_keepout > kMaxKeepout ||
        (n_keepout > 0 && !keepout_xy) || !(half >= 0.0))
        return SVSDF_ERR_INVALID;
    if (ctx->map_Z != 1) { ctx->err = "svsdf_extract_points: the map has several z layers, use svsdf_extract_points3d"; return SVSDF_ERR_INVALID; }
    // the flat case: one layer, every box spans it (centre z in the middle of the layer)
    std::vector<double> wp((size_t)W * 3);
    for (int w = 0; w < W; ++w) {
        wp[3 * (size_t)w] = waypoints_xy[2 * w];
        wp[3 * (size_t)w + 1] = waypoints_xy[2 * w + 1];
        wp[3 * (size_t)w + 2] = ctx->map_oz + 0.5 * ctx->map_res;
    }
    const double h3[3] = {half, half, half};
    return extract_impl(ctx, "svsdf_extract_points", wp.data(), W, h3, keepout_xy, n_keepout, clearance, n_points);
}

int svsdf_extract_points3d(svsdf_ctx *ctx, const double *waypoints_xyz, int W, const double *half_xyz, const double *keepout_xy,
                           int n_keepout, double clearance, int64_t *n_points) {
    if (!ctx || !waypoints_xyz || !half_xyz || W < 1 || W > kMaxWaypoints || n_keepout < 0 || n_keepout > kMaxKeepout ||
        (n_keepout > 0 && !keepout_xy) || !(half_xyz[0] >= 0.0) || !(half_xyz[1] >= 0.0) || !(half_xyz[2] >= 0.0))
        return SVSDF_ERR_INVALID;
    return extract_impl(ctx, "svsdf_extract_points3d", waypoints_xyz, W, half_xyz, keepout_xy, n_keepout, clearance, n_points);
}

}  // extern "C"
