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

#include "host/astar_flat.hpp"
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

// The neighbour loop of AstarPathSearcher::process (front_end_Astar.hpp:192-240) for ONE (node, neighbour cell), run by a whole warp
// (every lane passes the same arguments):
//   cond = isIndexValid(vi) && !isIndexOccupiedFlate(vi, 0) && checkKernelValue(fy, cy, vi) && checkSubSWCollision(state1, state2, aabb)
// The kernel test is the literal byte-wise one (all lanes in lockstep); the sub-swept-volume test (sw_manager.hpp:1171-1210)
// spreads the occupied cells of the box around the child (getPointsInAABB2D, PCSmap_manager.h:137-158) over the lanes,
// each lane walking the kt samples of its cell.  Returns the parts mask (bit 0 valid and free, bit 1 kernel test, bit 2
// sub-swept-volume test; the node passes iff it is 7) and the child yaw in cy.  Shared by k_expand_nodes and k_astar_search.
template <int SHAPE, bool XFORM>
__device__ __forceinline__ unsigned node_test(const ShapeParams &S, const FrontParams &F, const SubSwParams &P, const unsigned char *map,
                                              const unsigned char *kbytes, int ix, int iy, double fy, int nb, int lane, double &cy) {
    const int vx = ix + (nb / 3 - 1), vy = iy + (nb % 3 - 1);
    cy = fy;
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
    return parts;
}

// svsdf_front_expand: one warp per (node, neighbour cell)
template <int SHAPE, bool XFORM>
__global__ void __launch_bounds__(256) k_expand_nodes(const __grid_constant__ ShapeParams S, const __grid_constant__ FrontParams F,
                                                      const __grid_constant__ SubSwParams P, const unsigned char *map,
                                                      const unsigned char *kbytes, int64_t n, const int *node_ij, const double *node_yaw,
                                                      unsigned char *ok_out, double *child_yaw_out, unsigned char *parts_out) {
    const int lane = threadIdx.x & 31;
    const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= 9 * n) return;
    const int64_t q = w / 9;
    double cy;
    const unsigned parts = node_test<SHAPE, XFORM>(S, F, P, map, kbytes, node_ij[2 * q], node_ij[2 * q + 1], node_yaw[q], (int)(w % 9), lane, cy);
    if (lane == 0) {
        ok_out[w] = (parts == 7u) ? 1 : 0;
        child_yaw_out[w] = cy;
        if (parts_out) parts_out[w] = (unsigned char)parts;
    }
}

// svsdf_front_astar_device: whole searches, one CTA per search in flight (AstarPathSearch / getPath, front_end_Astar.hpp:243-390).
// Thread 0 runs the bookkeeping of host/astar_flat.hpp (pop, goal and budget tests, neighbour updates, path walk); the popped
// node goes through shared memory to the 9 warps, warp w tests neighbour w with node_test, and ok9 / yaw9 come back the same way.
// The grid is persistent and takes search indices from a global counter (reset by the host before the launch): no CTA waits
// for another, so nothing depends on how many CTAs are resident.  CTA b owns slot b of the pool: id int8, g / f / yaw double,
// father int32 and the heap, each NS + 1 long (NS = X * Y; slot NS is the start-node object).
//   * Only id[] is cleared (by the whole CTA) before each search: every other array is written before it is read (see FlatSearch).
//   * Heap capacity NS + 1 is enough: a slot is pushed only when its id goes from 0 (unseen) or -1 (closed) to 1 (open) and
//     leaves the heap when it is popped (id = -1), so each of the NS + 1 slots has at most one live entry; the start cell is marked
//     open but never pushed.  The overflow status (-1) stays as a guard.
//   * Every loop is bounded: the expansion loop by max_expansions + 1 pops (pop_next stops at the budget), the path walk by NS + 1.
constexpr int kAstarWarps = 9;

template <int SHAPE, bool XFORM>
__global__ void __launch_bounds__(kAstarWarps * 32, 2) k_astar_search(const __grid_constant__ ShapeParams S, const __grid_constant__ FrontParams F,
                                                                   const __grid_constant__ SubSwParams P, const unsigned char *map,
                                                                   const unsigned char *kbytes, const __grid_constant__ AstarArgs A) {
    __shared__ host::FlatSearch fs;  // thread 0's search state: in shared memory, so that it costs the node test no registers
    __shared__ int s_q, s_go, s_cx, s_cy;
    __shared__ double s_yaw;
    __shared__ unsigned char s_ok[9];
    __shared__ double s_cyaw[9];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int NS = F.X * F.Y;
    int8_t *id;
    {
        unsigned char *slot = A.pool + (size_t)blockIdx.x * A.slot_bytes;
        host::FlatHeapEntry *heap = reinterpret_cast<host::FlatHeapEntry *>(slot);
        double *g = reinterpret_cast<double *>(heap + (NS + 1));
        int32_t *father = reinterpret_cast<int32_t *>(g + 3 * (NS + 1));
        id = reinterpret_cast<int8_t *>(father + (NS + 1));
        if (tid == 0) {
            fs.X = F.X; fs.Y = F.Y; fs.NS = NS;
            fs.heap = heap; fs.heap_cap = NS + 1;
            fs.g = g; fs.f = g + (NS + 1); fs.yaw = g + 2 * (NS + 1);
            fs.father = father; fs.id = id;
        }
    }
    for (int round = 0; round < A.n; ++round) {  // a CTA runs at most n searches
        if (tid == 0) s_q = atomicAdd(A.next, 1);
        __syncthreads();
        const int q = s_q;
        if (q >= A.n) break;
        const int4 c = reinterpret_cast<const int4 *>(A.cells)[q];
        if (c.x < 0) {  // start or goal outside the map (isInMap): the search does not run
            if (tid == 0) { A.len[q] = 0; A.expansions[q] = 0; A.status[q] = 0; }
            __syncthreads();
            continue;
        }
        for (int i = tid; i <= NS; i += blockDim.x) id[i] = 0;
        __syncthreads();
        if (tid == 0) fs.begin(c.x, c.y, c.z, c.w);
        for (int64_t it = 0; it <= A.max_expansions; ++it) {
            if (tid == 0) {
                int cx = 0, cy = 0;
                double cyaw = 0.0;
                s_go = fs.pop_next(A.max_expansions, cx, cy, cyaw) ? 1 : 0;
                s_cx = cx; s_cy = cy; s_yaw = cyaw;
            }
            __syncthreads();
            if (!s_go) break;
            {
                double cyw;
                const unsigned parts = node_test<SHAPE, XFORM>(S, F, P, map, kbytes, s_cx, s_cy, s_yaw, warp, lane, cyw);
                if (lane == 0) { s_ok[warp] = (parts == 7u) ? 1 : 0; s_cyaw[warp] = cyw; }
            }
            __syncthreads();
            if (tid == 0) fs.apply(s_cx, s_cy, s_ok, s_cyaw);
        }
        if (tid == 0) {
            int st = fs.status == 0 ? -1 : fs.status, len = 0;  // still running after max_expansions + 1 pops: cannot happen
            if (st == 1) {
                const int np = fs.path(F.ox, F.oy, F.map_res, A.max_path, A.paths + (size_t)q * A.max_path * 3);
                if (np < 0) st = -1;
                else if (np > A.max_path) st = 4;
                else len = np;
            }
            A.len[q] = len; A.expansions[q] = (int)fs.expansions; A.status[q] = st;
        }
        __syncthreads();  // the next search clears this slot's id[] only after thread 0 is done with it
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

// grid <= 0: only report the resident CTAs per SM (occupancy query) in *ctas_per_sm
template <int SHAPE, bool XFORM>
cudaError_t launch_astar_t(const ShapeParams &S, const FrontParams &F, const SubSwParams &P, const unsigned char *map, const unsigned char *kbytes,
                           const AstarArgs &A, int grid, int *ctas_per_sm, cudaStream_t st) {
    if (grid <= 0) return cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas_per_sm, k_astar_search<SHAPE, XFORM>, kAstarWarps * 32, 0);
    k_astar_search<SHAPE, XFORM><<<grid, kAstarWarps * 32, 0, st>>>(S, F, P, map, kbytes, A);
    return cudaGetLastError();
}

}  // namespace

// The analytic functors the front end is defined for; Polygon / mesh: the reference defines no rotated kernels for them
#define SVSDF_FRONT_SHAPES(CASE)                                                                                                 \
    CASE(SH_STAR) CASE(SH_HORSESHOE) CASE(SH_PIE) CASE(SH_PIE2) CASE(SH_ARC) CASE(SH_TUNNEL) CASE(SH_CUTDISK) CASE(SH_TRAPEZOID) \
    CASE(SH_RHOMBUS) CASE(SH_HEART) CASE(SH_ROUNDEDX) CASE(SH_BIGX) CASE(SH_ROUNDEDCROSS) CASE(SH_VESICA) CASE(SH_MOON)         \
    CASE(SH_UNEVENCAPSULE) CASE(SH_CIRCLE)

cudaError_t launch_front_cells(const ShapeParams &S, const FrontParams &F, const double *yaws, unsigned char *cells, cudaStream_t st) {
    switch (S.id) {
#define SVSDF_CASE(ID) \
    case ID: return S.has_xform ? launch_cells_t<ID, true>(S, F, yaws, cells, st) : launch_cells_t<ID, false>(S, F, yaws, cells, st);
        SVSDF_FRONT_SHAPES(SVSDF_CASE)
#undef SVSDF_CASE
        default: return cudaErrorInvalidValue;
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
        SVSDF_FRONT_SHAPES(SVSDF_CASE)
#undef SVSDF_CASE
        default: return cudaErrorInvalidValue;
    }
}

cudaError_t launch_front_astar(const ShapeParams &S, const FrontParams &F, const SubSwParams &P, const unsigned char *map,
                               const unsigned char *kbytes, const AstarArgs &A, int grid, int *ctas_per_sm, cudaStream_t st) {
    switch (S.id) {
#define SVSDF_CASE(ID)                                                                                            \
    case ID:                                                                                                      \
        return S.has_xform ? launch_astar_t<ID, true>(S, F, P, map, kbytes, A, grid, ctas_per_sm, st)             \
                           : launch_astar_t<ID, false>(S, F, P, map, kbytes, A, grid, ctas_per_sm, st);
        SVSDF_FRONT_SHAPES(SVSDF_CASE)
#undef SVSDF_CASE
        default: return cudaErrorInvalidValue;
    }
}
#undef SVSDF_FRONT_SHAPES

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
