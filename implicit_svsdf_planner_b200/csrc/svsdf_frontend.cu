// svsdf_frontend.cu — K5: the collision kernels of the reference's A* front end on the device (SURVEY.md §8f rank 3).
//
// Reference (paths relative to the reference project's src/):
//   BasicShape::initShape                 utils/include/utils/Shape.hpp:386-430   yaw-indexed occupancy kernels of the robot shape:
//                                         cell (a, b) of kernel k is set iff getonlySDF((x_a, y_b, 0), Rz(yaw_k)) <= safemargin
//   getonlySDF(pos_rel, R_obj)            Shape.hpp:481-485 ... (every analytic class): ((p - trans) * Rotate * R_obj).head(2)
//   byteShapeKernel::generateByteKernel   Shape.hpp:194-216  (MSB-first rows, or_mask)
//   SweptVolumeManager::kernelConv<true>  swept_volume/include/swept_volume/sw_manager.hpp:1068-1095: byte-AND of the shape's byte
//                                         kernel with the window of the inflated, byte-packed map kernel (generateMapKernel2D)
//   visit_kernels_by_distance, checkKernelValue   sw_manager.hpp:1099-1169
//
// GPU formulation.  The A* calls kernelConv once per (expanded cell, yaw) — 51 byte operations each, latency bound on
// the host.  Here the whole configuration-space obstacle map is produced in one pass instead: free[k][x][y] for every yaw
// kernel k and every cell, 32 cells (one output word) per thread, each kernel row applied as shifted ORs of the two map
// words under it (funnel shifts; the map's MSB-first bit order is kept so the words are the map's own bytes).  Integer
// work on an L2-resident input (the packed map is X*Y/8 bytes); output K*X*Y/8 bytes — after that a collision test is
// one bit lookup.  k_check_kernel_value restates the per-node test literally (byte by byte) on top of the same data and
// is what the tests compare the word-parallel kernel with.
#include <cuda_runtime.h>
#include <stdint.h>

#include "svsdf_shapes.cuh"
#include "svsdf_types.h"

namespace svsdf {

namespace {

template <int SHAPE, bool XFORM>
__global__ void __launch_bounds__(256) k_shape_kernel_cells(const __grid_constant__ ShapeParams S, FrontParams F,
                                                            const double *yaws, unsigned char *cells) {
    const int ks = F.kernel_size;
    const int n = F.kernel_count * ks * ks;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    const int k = idx / (ks * ks), a = (idx / ks) % ks, b = idx % ks;
    double s, c;
    dev::sincos_portable(yaws[k], s, c);
    const int size_side = (int)(0.5 * (ks - 1));
    const double x = F.res * a - size_side * F.res;  // Shape.hpp:413-414
    const double y = F.res * b - size_side * F.res;
    double w0 = x, w1 = y;
    if (XFORM) {
        const double v0 = x - S.trans[0], v1 = y - S.trans[1];
        w0 = v0 * S.rot[0] + v1 * S.rot[2];
        w1 = v0 * S.rot[1] + v1 * S.rot[3];
    }
    const double u0 = w0 * c + w1 * s;      // R_obj = [[c, -s], [s, c]], row vector on the left
    const double u1 = w0 * (-s) + w1 * c;
    const double sdf = dev::ShapeFn<SHAPE>::sdf(S, u0, u1);
    cells[idx] = (sdf <= F.safemargin) ? 1 : 0;
}

// 32 consecutive map bits of inflated row `row`, starting at inflated column 32 * w, MSB = lowest column
__device__ __forceinline__ unsigned map_word(const unsigned char *row, int row_bytes, int w) {
    const int b0 = 4 * w;
    unsigned v = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q)
        if (b0 + q < row_bytes) v |= (unsigned)__ldg(row + b0 + q) << (24 - 8 * q);
    return v;
}

// out[k][x][yw]: bit (31 - t) of the word <-> cell y = 32 * yw + t; 1 = kernelConv(k, (x, y)) is true (free)
__global__ void __launch_bounds__(256) k_cspace(FrontParams F, const unsigned char *map, const unsigned *rowmask, unsigned *out) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int W = F.out_words;
    const int64_t n = (int64_t)F.kernel_count * F.X * W;
    if (idx >= n) return;
    const int yw = (int)(idx % W), x = (int)((idx / W) % F.X), k = (int)(idx / ((int64_t)W * F.X));
    const unsigned *rm = rowmask + k * F.kernel_size;
    unsigned coll = 0u;
    for (int i = 0; i < F.kernel_size; ++i) {
        unsigned m = rm[i];
        if (m == 0u) continue;
        const unsigned char *row = map + (int64_t)(x + i) * F.row_bytes;  // window rows start at inflated row x
        const unsigned w0 = map_word(row, F.row_bytes, yw), w1 = map_word(row, F.row_bytes, yw + 1);
        while (m) {
            const int j = __clz(m);  // kernel column j (MSB first)
            m &= ~(0x80000000u >> j);
            coll |= __funnelshift_l(w1, w0, j);  // map bits at columns (y + j) for the 32 cells of this word
        }
    }
    unsigned fr = ~coll;
    const int y0 = 32 * yw;
    if (y0 + 32 > F.Y) fr &= (F.Y - y0 >= 32) ? 0xffffffffu : ~(0xffffffffu >> (F.Y - y0));  // cells beyond Y: not free
    out[idx] = fr;
}

// kernelConv<true>, literally (sw_manager.hpp:1068-1095)
__device__ __forceinline__ bool kernel_conv_byte(const FrontParams &F, const unsigned char *map, const unsigned char *kbytes, int kernel_i,
                                                 int ind_x, int ind_y) {
    const int bpr = (F.kernel_size + 7) / 8;
    const int64_t total = (int64_t)(F.X + 2 * F.h) * F.row_bytes;
    for (int i = 0; i < F.kernel_size; i++) {
        const int64_t start = (int64_t)(ind_x + i) * F.row_bytes + (ind_y / 8);
        const int off = ind_y % 8;
        for (int j = 0; j < bpr; j++) {
            const unsigned m0 = (start + j < total) ? __ldg(map + start + j) : 0u;
            const unsigned m1 = (start + j + 1 < total) ? __ldg(map + start + j + 1) : 0u;
            const unsigned block = ((m0 << off) | (m1 >> (8 - off))) & 0xffu;
            if (kbytes[((int64_t)kernel_i * F.kernel_size + i) * bpr + j] & block) return false;
        }
    }
    return true;
}

__global__ void __launch_bounds__(128) k_check_kernel_value(FrontParams F, const unsigned char *map, const unsigned char *kbytes, int64_t n,
                                                            const double *father_yaw, const int *ind_xy, unsigned char *ok_out,
                                                            double *child_yaw_out) {
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n) return;
    const double pi = 3.1415926536;  // sw_manager.hpp:20
    const int count = F.kernel_count;
    const double fy = father_yaw[q];
    int father_i = int(count * ((fy + pi) / (2 * pi)));
    father_i = father_i < 0 ? 0 : (father_i >= count ? count - 1 : father_i);
    const int ix = ind_xy[2 * q], iy = ind_xy[2 * q + 1];
    // visit_kernels_by_distance: breadth-first over the yaw ring, at most maxdeepth + 1 = 11 kernels
    unsigned long long visited = 1ull << father_i;
    int queue[24];
    int head = 0, tail = 0, deep = 0;
    queue[tail++] = father_i;
    bool ok = false;
    int ret = father_i;
    while (head < tail) {
        deep++;
        const int x = queue[head++];
        if (kernel_conv_byte(F, map, kbytes, x, ix, iy)) { ret = x; ok = true; break; }
#pragma unroll
        for (int d = 0; d < 2; ++d) {
            int nx = x + (d == 0 ? -1 : 1);
            if (nx < 0) nx = count - 1;
            if (nx >= count) nx = 0;
            if ((visited >> nx) & 1ull) continue;
            visited |= 1ull << nx;
            if (tail < 24) queue[tail++] = nx;
        }
        if (deep > 10) break;
    }
    ok_out[q] = ok ? 1 : 0;
    child_yaw_out[q] = ok ? (2 * pi * (ret) / count - pi) : fy;
}

__device__ __forceinline__ bool map_occupied(const FrontParams &F, const unsigned char *map, int i, int j) {
    const int c = j + F.h;
    return (__ldg(map + (int64_t)(i + F.h) * F.row_bytes + (c >> 3)) & (0x80u >> (c & 7))) != 0;
}

// GridMap3D::getGridIndex after projInMap (Gridmap3D.cpp:137-172, PCSmap_manager.h:126-133), one axis
__device__ __forceinline__ int grid_index_1d(double p, double lo, double hi, double res, int size) {
    if (p < lo) p = lo;
    if (p > hi) p = hi;
    int i = (int)floor((p - lo) / res);
    if (i < 0) i = 0;
    if (i >= size) i = size - 1;
    return i;
}

// The neighbour loop of AstarPathSearcher::process (front_end_Astar.hpp:192-240), one warp per (node, neighbour cell):
//   cond = isIndexValid(vi) && !isIndexOccupiedFlate(vi, 0) && checkKernelValue(fy, cy, vi) && checkSubSWCollision(state1, state2, aabb)
// The kernel test is the literal byte-wise one (all lanes in lockstep); the sub-swept-volume test (sw_manager.hpp:1171-1210)
// spreads the occupied cells of the box around the child (getPointsInAABB2D, PCSmap_manager.h:137-158) over the lanes,
// each lane walking the kt samples of its cell.
template <int SHAPE, bool XFORM>
__global__ void __launch_bounds__(256) k_expand_nodes(const __grid_constant__ ShapeParams S, const __grid_constant__ FrontParams F,
                                                      const __grid_constant__ SubSwParams P, const unsigned char *map,
                                                      const unsigned char *kbytes, int64_t n, const int *node_ij, const double *node_yaw,
                                                      unsigned char *ok_out, double *child_yaw_out, unsigned char *parts_out) {
    const int lane = threadIdx.x & 31;
    const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= 9 * n) return;
    const int64_t q = w / 9;
    const int nb = (int)(w % 9);
    const int ix = node_ij[2 * q], iy = node_ij[2 * q + 1];
    const int vx = ix + (nb / 3 - 1), vy = iy + (nb % 3 - 1);
    const double fy = node_yaw[q];
    double cy = fy;
    unsigned parts = 0;
    const bool valid = vx >= 0 && vx < F.X && vy >= 0 && vy < F.Y;
    if (valid) {
        if (!map_occupied(F, map, vx, vy)) parts |= 1u;
        // checkKernelValue (sw_manager.hpp:1158-1169) -> visit_kernels_by_distance (:1099-1156)
        {
            const double pi = 3.1415926536;
            const int count = F.kernel_count;
            int father_i = int(count * ((fy + pi) / (2 * pi)));
            father_i = father_i < 0 ? 0 : (father_i >= count ? count - 1 : father_i);
            unsigned long long visited = 1ull << father_i;
            int queue[24];
            int head = 0, tail = 0, deep = 0;
            queue[tail++] = father_i;
            while (head < tail) {
                deep++;
                const int x = queue[head++];
                if (kernel_conv_byte(F, map, kbytes, x, vx, vy)) {
                    cy = 2 * pi * (x) / count - pi;
                    parts |= 2u;
                    break;
                }
#pragma unroll
                for (int d = 0; d < 2; ++d) {
                    int nx = x + (d == 0 ? -1 : 1);
                    if (nx < 0) nx = count - 1;
                    if (nx >= count) nx = 0;
                    if ((visited >> nx) & 1ull) continue;
                    visited |= 1ull << nx;
                    if (tail < 24) queue[tail++] = nx;
                }
                if (deep > 10) break;
            }
        }
        // checkSubSWCollision(state1 = (father centre, fy), state2 = (child centre, cy), points in the box around the child)
        const double f0 = (ix + 0.5) * F.map_res + F.ox, f1 = (iy + 0.5) * F.map_res + F.oy;
        const double c0 = (vx + 0.5) * F.map_res + F.ox, c1 = (vy + 0.5) * F.map_res + F.oy;
        const double xmax = F.ox + F.X * F.map_res, ymax = F.oy + F.Y * F.map_res;
        const int i1 = grid_index_1d(c0 - P.half_box, F.ox, xmax, F.map_res, F.X), i2 = grid_index_1d(c0 + P.half_box, F.ox, xmax, F.map_res, F.X);
        const int j1 = grid_index_1d(c1 - P.half_box, F.oy, ymax, F.map_res, F.Y), j2 = grid_index_1d(c1 + P.half_box, F.oy, ymax, F.map_res, F.Y);
        const int nj = j2 - j1 + 1, cells = (i2 - i1 + 1) * nj;
        // occupied cells are found 32 at a time (ballot); for each one the kt samples are spread over the lanes (2 per lane at
        // 51 samples), so the latency of an edge is ~2 evaluations per obstacle cell instead of 51 per lane.  The test is
        // a plain "any sample inside the shape", so the order does not matter.
        bool hit = false;
        for (int base = 0; base < cells && !hit; base += 32) {
            const int c = base + lane;
            bool occ = false;
            if (c < cells) occ = map_occupied(F, map, i1 + c / nj, j1 + c % nj);
            unsigned m = __ballot_sync(0xffffffffu, occ);
            while (m && !hit) {
                const int b = __ffs(m) - 1;
                m &= m - 1;
                const int cc = base + b;
                const int i = i1 + cc / nj, j = j1 + cc % nj;
                const double px = (i + 0.5) * F.map_res + F.ox, py = (j + 0.5) * F.map_res + F.oy;
                bool mine = false;
                for (int t = lane; t < P.nkt && !mine; t += 32) {
                    const double kt = P.kt[t], om = 1 - kt;
                    const double lx = kt * c0 + om * f0, ly = kt * c1 + om * f1, yaw = kt * cy + om * fy;
                    double sn, cs;
                    dev::sincos_portable(yaw, sn, cs);
                    const double d0 = px - lx, d1 = py - ly;
                    const double rx = cs * d0 + sn * d1, ry = -sn * d0 + cs * d1;
                    mine = dev::shape_sdf<SHAPE, XFORM>(S, rx, ry) < 0;
                }
                hit = __any_sync(0xffffffffu, mine);
            }
        }
        if (!hit) parts |= 4u;
    }
    if (lane == 0) {
        ok_out[w] = (parts == 7u) ? 1 : 0;
        child_yaw_out[w] = cy;
        if (parts_out) parts_out[w] = (unsigned char)parts;
    }
}

template <int SHAPE, bool XFORM>
cudaError_t launch_expand_t(const ShapeParams &S, const FrontParams &F, const SubSwParams &P, const unsigned char *map, const unsigned char *kbytes,
                            int64_t n, const int *node_ij, const double *node_yaw, unsigned char *ok_out, double *child_yaw_out,
                            unsigned char *parts_out, cudaStream_t st) {
    const int64_t threads = 9 * n * 32;
    k_expand_nodes<SHAPE, XFORM><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(S, F, P, map, kbytes, n, node_ij, node_yaw, ok_out,
                                                                                     child_yaw_out, parts_out);
    return cudaGetLastError();
}

template <int SHAPE, bool XFORM>
cudaError_t launch_cells_t(const ShapeParams &S, const FrontParams &F, const double *yaws, unsigned char *cells, cudaStream_t st) {
    const int n = F.kernel_count * F.kernel_size * F.kernel_size;
    k_shape_kernel_cells<SHAPE, XFORM><<<(n + 255) / 256, 256, 0, st>>>(S, F, yaws, cells);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_front_cells(const ShapeParams &S, const FrontParams &F, const double *yaws, unsigned char *cells, cudaStream_t st) {
    switch (S.id) {
#define SVSDF_CASE(ID) \
    case ID: return S.has_xform ? launch_cells_t<ID, true>(S, F, yaws, cells, st) : launch_cells_t<ID, false>(S, F, yaws, cells, st);
        SVSDF_CASE(SH_STAR)
        SVSDF_CASE(SH_HORSESHOE)
        SVSDF_CASE(SH_PIE)
        SVSDF_CASE(SH_PIE2)
        SVSDF_CASE(SH_ARC)
        SVSDF_CASE(SH_TUNNEL)
        SVSDF_CASE(SH_CUTDISK)
        SVSDF_CASE(SH_TRAPEZOID)
        SVSDF_CASE(SH_RHOMBUS)
        SVSDF_CASE(SH_HEART)
        SVSDF_CASE(SH_ROUNDEDX)
        SVSDF_CASE(SH_BIGX)
        SVSDF_CASE(SH_ROUNDEDCROSS)
        SVSDF_CASE(SH_VESICA)
        SVSDF_CASE(SH_MOON)
        SVSDF_CASE(SH_UNEVENCAPSULE)
        SVSDF_CASE(SH_CIRCLE)
#undef SVSDF_CASE
        default: return cudaErrorInvalidValue;  // Polygon / mesh: the reference defines no rotated kernels for them
    }
}

cudaError_t launch_front_expand(const ShapeParams &S, const FrontParams &F, const SubSwParams &P, const unsigned char *map,
                                const unsigned char *kbytes, int64_t n, const int *node_ij, const double *node_yaw, unsigned char *ok_out,
                                double *child_yaw_out, unsigned char *parts_out, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    switch (S.id) {
#define SVSDF_CASE(ID)                                                                                                              \
    case ID:                                                                                                                        \
        return S.has_xform ? launch_expand_t<ID, true>(S, F, P, map, kbytes, n, node_ij, node_yaw, ok_out, child_yaw_out, parts_out, st) \
                           : launch_expand_t<ID, false>(S, F, P, map, kbytes, n, node_ij, node_yaw, ok_out, child_yaw_out, parts_out, st);
        SVSDF_CASE(SH_STAR)
        SVSDF_CASE(SH_HORSESHOE)
        SVSDF_CASE(SH_PIE)
        SVSDF_CASE(SH_PIE2)
        SVSDF_CASE(SH_ARC)
        SVSDF_CASE(SH_TUNNEL)
        SVSDF_CASE(SH_CUTDISK)
        SVSDF_CASE(SH_TRAPEZOID)
        SVSDF_CASE(SH_RHOMBUS)
        SVSDF_CASE(SH_HEART)
        SVSDF_CASE(SH_ROUNDEDX)
        SVSDF_CASE(SH_BIGX)
        SVSDF_CASE(SH_ROUNDEDCROSS)
        SVSDF_CASE(SH_VESICA)
        SVSDF_CASE(SH_MOON)
        SVSDF_CASE(SH_UNEVENCAPSULE)
        SVSDF_CASE(SH_CIRCLE)
#undef SVSDF_CASE
        default: return cudaErrorInvalidValue;
    }
}

cudaError_t launch_front_cspace(const FrontParams &F, const unsigned char *map, const unsigned *rowmask, unsigned *out, cudaStream_t st) {
    const int64_t n = (int64_t)F.kernel_count * F.X * F.out_words;
    if (n == 0) return cudaSuccess;
    k_cspace<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(F, map, rowmask, out);
    return cudaGetLastError();
}

cudaError_t launch_front_check(const FrontParams &F, const unsigned char *map, const unsigned char *kbytes, int64_t n, const double *father_yaw,
                               const int *ind_xy, unsigned char *ok_out, double *child_yaw_out, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    k_check_kernel_value<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(F, map, kbytes, n, father_yaw, ind_xy, ok_out, child_yaw_out);
    return cudaGetLastError();
}

}  // namespace svsdf
