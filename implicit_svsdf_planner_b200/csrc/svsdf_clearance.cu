// svsdf_clearance.cu — the band of occupied map columns that svsdf_map_clearance evaluates (contract: include/svsdf.h, DESIGN.md §7).
// Compiled with -fmad=false: a cell centre is ((i + 0.5) res + ox, (j + 0.5) res + oy) rounded as k_extract_write rounds it, so the
// points are bit for bit the ones svsdf_extract_points[3d] hands the back end.
//
// Pipeline (the host side is clearance_bands in svsdf_runtime_swept.cpp; svsdf_map_clearance is its one-trajectory case):
//   k_cl_count   the words of every problem's reach rectangle, one item per 32-cell word, row-major, padded to whole CTAs of 256
//                (the CTAs of problem k follow those of problem k - 1, so the CTA order is problem order, then map order).  The
//                problem's samples whose reach touches the CTA's cell-centre box go to a shared list; each item ORs its word over
//                the z layers (a column is occupied when any layer is) and keeps the set bits whose centre lies within some listed
//                sample's reach.  Writes the band bits and the CTA's band count.  A last segment covers the whole map and only
//                counts its occupied columns.
//   k_sw_scan    exclusive prefix of the per-CTA counts (svsdf_swept.cu, one CTA).
//   k_cl_write   the band's cells (i, j) and centres, concatenated in problem order, each in map order, into the clearance's own
//                point buffer.
//   (then svsdf_query's kernels for one trajectory, the multi-problem kernels of svsdf_kernels_multi.cuh for n)
#include <cuda_runtime.h>
#include <stdint.h>

#include "svsdf_launch.h"
#include "svsdf_types.h"

namespace svsdf {
namespace {

// exclusive prefix over the 256 threads of a CTA; *total = the CTA's sum.  s_w: 8 ints of shared memory, one array per concurrent use.
__device__ __forceinline__ int block_scan256(int v, int *s_w, int *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_w[warp] = x;
    __syncthreads();
    int before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
        const int s = s_w[w];
        if (w < warp) before += s;
        all += s;
    }
    __syncthreads();
    *total = all;
    return before + x - v;
}

__device__ __forceinline__ unsigned interval_mask(int lo, int hi) {  // bits lo..hi (inclusive) of a 32-bit word
    lo = lo < 0 ? 0 : lo;
    hi = hi > 31 ? 31 : hi;
    if (lo > hi) return 0u;
    return (0xffffffffu >> (31 - hi)) & (0xffffffffu << lo);
}

// getGridCubeCenter: (idx + 0.5) * res + min, as k_extract_write computes it
__device__ __forceinline__ double centre_x(const ClearanceArgs &A, int i) { return ((double)i + 0.5) * A.res + A.ox; }
__device__ __forceinline__ double centre_y(const ClearanceArgs &A, int j) { return ((double)j + 0.5) * A.res + A.oy; }

// Word wy of map row i (bit k <-> padded y = 32 wy + k) ORed over the z layers, restricted to real cells (0 <= y < Y): the padding of
// the map kernel is not an obstacle here.  The bytes are MSB first (or_mask = {0x80 .. 0x01}); reversing the bits of every byte
// commutes with the OR, so it is done once.
__device__ __forceinline__ unsigned column_word(const ClearanceArgs &A, int i, int wy) {
    const int b0 = 4 * wy;
    unsigned w = 0;
    for (int z = 0; z < A.Z; ++z) {
        const unsigned char *row = A.map + (int64_t)z * A.layer + (int64_t)(i + A.h) * A.row_bytes;
#pragma unroll
        for (int q = 0; q < 4; ++q)
            if (b0 + q < A.row_bytes) w |= (unsigned)row[b0 + q] << (8 * q);
    }
    w = __byte_perm(__brev(w), 0, 0x0123);
    return w & interval_mask(A.h - 32 * wy, A.h + A.Y - 1 - 32 * wy);
}

// The items of this CTA in problem C's rectangle: item t = first + threadIdx.x (< n_items) is word wy0 + t % nW of row i0 + t / nW.
// Returns the item's band bits (its occupied columns whose centre lies within some sample's reach; all of them when `all`) and its
// occupied bits in *occ.
__device__ __forceinline__ unsigned cta_band(const ClearanceArgs &A, const ClearanceProblem &C, int64_t first, int *s_list, int *s_n,
                                             unsigned *occ_out) {
    const double *samp = A.samp + 3 * (int64_t)C.samp0;
    const int64_t last = min(first + (int64_t)blockDim.x - 1, C.n_items - 1);
    const int64_t t = first + threadIdx.x;
    int i = 0, wy = 0;
    unsigned occ = 0u;
    if (t < C.n_items) {
        i = C.i0 + (int)(t / C.nW);
        wy = C.wy0 + (int)(t % C.nW);
        occ = column_word(A, i, wy);
    }
    *occ_out = occ;
    unsigned band = C.all ? occ : 0u;
    if (!C.all) {  // uniform over the CTA
        // box of the CTA's cell centres: its rows, and the y range of its words when it lies in one row (the whole map's otherwise)
        const int i0 = C.i0 + (int)(first / C.nW), i1 = C.i0 + (int)(last / C.nW);
        int j0 = 0, j1 = A.Y - 1;
        if (i0 == i1) {
            j0 = max(32 * (C.wy0 + (int)(first % C.nW)) - A.h, 0);
            j1 = min(32 * (C.wy0 + (int)(last % C.nW)) + 31 - A.h, A.Y - 1);
        }
        const double bx0 = centre_x(A, i0), bx1 = centre_x(A, i1), by0 = centre_y(A, j0), by1 = centre_y(A, j1);
        if (threadIdx.x == 0) *s_n = 0;
        __syncthreads();
        // a sample that reaches a centre of the CTA reaches its box: the centres are monotone in the index and the rounded differences
        // and squares are monotone, so the box distance is never larger than the centre distance computed below (k_sw_classify's test)
        for (int k = threadIdx.x; k < C.n_samp; k += blockDim.x) {
            const double sx = samp[3 * k], sy = samp[3 * k + 1], r = samp[3 * k + 2];
            const double dx = fmax(fmax(bx0 - sx, sx - bx1), 0.0), dy = fmax(fmax(by0 - sy, sy - by1), 0.0);
            if (dx * dx + dy * dy <= r * r) s_list[atomicAdd(s_n, 1)] = k;
        }
        __syncthreads();
        const int n = *s_n;
        if (occ && n) {
            const double cx = centre_x(A, i);
            const int ybase = 32 * wy - A.h;
            for (unsigned bits = occ; bits; bits &= bits - 1) {
                const int k = __ffs(bits) - 1;
                const double cy = centre_y(A, ybase + k);
                bool in = false;
                for (int q = 0; q < n && !in; ++q) {
                    const int s = s_list[q];
                    const double dx = cx - samp[3 * s], dy = cy - samp[3 * s + 1], r = samp[3 * s + 2];
                    in = dx * dx + dy * dy <= r * r;
                }
                if (in) band |= 1u << k;
            }
        }
    }
    return band;
}

// the band cells of word wy of row i, from list position pos on
__device__ __forceinline__ void write_cells(const ClearanceArgs &A, unsigned band, int i, int wy, int64_t pos) {
    const int ybase = 32 * wy - A.h;
    const double cx = centre_x(A, i);
    for (; band; band &= band - 1) {
        const int j = ybase + __ffs(band) - 1;
        A.ij[2 * pos] = i;
        A.ij[2 * pos + 1] = j;
        A.pts[2 * pos] = cx;
        A.pts[2 * pos + 1] = centre_y(A, j);
        ++pos;
    }
}

// The CTAs of problem k are cta0[k] .. cta0[k + 1] - 1, in problem order; the last segment counts the occupied columns of the whole
// map and has no band.  Items: one per (CTA, thread), so band[] is indexed by blockIdx.x * 256 + threadIdx.x.
__device__ __forceinline__ const ClearanceProblem &cta_problem(const ClearanceArgs &A) {
    int lo = 0, hi = A.n_prob - 1;  // the last k with cta0 <= blockIdx.x (a problem without CTAs shares cta0 with the next one)
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (A.prob[mid].cta0 <= (int64_t)blockIdx.x) lo = mid;
        else hi = mid - 1;
    }
    return A.prob[lo];
}

__global__ void __launch_bounds__(256) k_cl_count(const __grid_constant__ ClearanceArgs A) {
    __shared__ int s_list[kSweptMaxSamples];
    __shared__ int s_n;
    __shared__ int s_w[2][8];
    const ClearanceProblem &pr = cta_problem(A);
    unsigned occ;
    unsigned band = cta_band(A, pr, ((int64_t)blockIdx.x - pr.cta0) * blockDim.x, s_list, &s_n, &occ);
    if (pr.occ_only) band = 0u;
    else occ = 0u;
    A.band[(int64_t)blockIdx.x * blockDim.x + threadIdx.x] = band;
    int n_band, n_occ;
    block_scan256(__popc(band), s_w[0], &n_band);
    block_scan256(__popc(occ), s_w[1], &n_occ);
    if (threadIdx.x == 0) {
        A.blk[blockIdx.x] = n_band;
        if (n_occ) atomicAdd(A.n_occ, (unsigned long long)n_occ);  // integer sum: the same total in any order
    }
}

__global__ void __launch_bounds__(256) k_cl_write(const __grid_constant__ ClearanceArgs A) {
    __shared__ int s_w[8];
    const unsigned band = A.band[(int64_t)blockIdx.x * blockDim.x + threadIdx.x];
    int total;
    const int64_t pos = (int64_t)A.blk[blockIdx.x] + block_scan256(__popc(band), s_w, &total);
    if (!band) return;
    const ClearanceProblem &pr = cta_problem(A);
    const int64_t t = ((int64_t)blockIdx.x - pr.cta0) * blockDim.x + threadIdx.x;
    write_cells(A, band, pr.i0 + (int)(t / pr.nW), pr.wy0 + (int)(t % pr.nW), pos);
}

}  // namespace

cudaError_t launch_clearance(int what, const ClearanceArgs &A, cudaStream_t st) {
    const unsigned nblk = (unsigned)((A.n_items + 255) / 256);
    switch (what) {
        case 0: k_cl_count<<<nblk, 256, 0, st>>>(A); break;
        case 1: k_cl_write<<<nblk, 256, 0, st>>>(A); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

}  // namespace svsdf
