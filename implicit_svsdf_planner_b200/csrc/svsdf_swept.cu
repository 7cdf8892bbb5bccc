// svsdf_swept.cu — the narrow-band marching-squares mesher of svsdf_swept_contour and svsdf_swept_contour_multi (contract:
// include/svsdf.h, DESIGN.md §7).  Compiled with -fmad=false, and every operation that makes a vertex is an explicit _rn intrinsic: the
// vertices depend on the field only, whichever build (strict or fast) evaluated it.
//
// Every kernel runs over the concatenation of n problems (SweptProblem; the single call is n = 1): a CTA finds its problem by a binary
// search of the table and works on that problem's grid (Grid) exactly as it would alone.  Problem k owns whole marching-squares blocks,
// so its corners, counts and outputs are contiguous and in problem order, and one k_sw_scan gives every problem its own prefix.
//
// Pipeline (the host side is swept_run in svsdf_runtime_swept.cpp):
//   k_sw_classify  one CTA per 16 x 16 tile: the path samples whose reach touches the tile's 18 x 18 corner region go to a shared list;
//                  each region corner is tested against that list only (unproven: within some sample's reach); a corner is needed
//                  when one of the cells around it has an unproven corner.  Writes the need flags, NaN into the field, the tile's count
//                  and adds it to the problem's needed corners.
//   k_sw_scan      exclusive prefix of per-CTA counts (one CTA).
//   k_sw_compact   the needed corners, tile by tile, into the mesher's own point buffer (x, y) and their corner indices.
//   (the outer solve of svsdf_query runs on that buffer: one problem's kernels, or the multi-problem ones for n problems)
//   k_sw_scatter   the values into the field.
//   k_sw_count     per corner: crossing horizontal / vertical edge, inside corner; per cell: segments and triangles.  Per-CTA sums, the
//                  problem's totals, its non-finite and clipped flags.
//   k_sw_vertices  vertex coordinates and the (problem-local) vertex id of every crossing edge and inside corner.
//   k_sw_cells     segments and triangles.
#include <cuda_runtime.h>

#include <cmath>

#include "svsdf_launch.h"
#include "svsdf_types.h"

namespace svsdf {
namespace {

constexpr int kReg = kSweptTile + 2;  // corner region of a tile: one corner of halo on each side

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

// The problem owning tile / block x of the concatenation: the last k with tile0 (by_block: blk0) <= x.
__device__ __forceinline__ int find_problem(const SweptArgs &A, int64_t x, bool by_block) {
    int lo = 0, hi = A.n_prob - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if ((by_block ? A.prob[mid].blk0 : A.prob[mid].tile0) <= x) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// One problem's grid: its lattice origin and size, and its corners' need flags, field and vertex ids (from corner kSweptBlock * blk0).
struct Grid {
    int64_t i0, j0;
    int nx, ny;
    double h, iso;
    unsigned char *need;
    double *field;
    int *vid;
};
__device__ __forceinline__ Grid grid_of(const SweptArgs &A, const SweptProblem &p) {
    const int64_t c0 = (int64_t)kSweptBlock * p.blk0;
    return Grid{p.i0, p.j0, p.nx, p.ny, A.h, A.iso, A.need + c0, A.field + c0, A.vid + 3 * c0};
}

__device__ __forceinline__ double corner_x(const Grid &G, int64_t a) { return __dmul_rn((double)(G.i0 + a), G.h); }
__device__ __forceinline__ double corner_y(const Grid &G, int64_t b) { return __dmul_rn((double)(G.j0 + b), G.h); }

__global__ void __launch_bounds__(256) k_sw_classify(SweptArgs A) {
    __shared__ int s_list[kSweptMaxSamples];
    __shared__ int s_n;
    __shared__ unsigned char s_unp[kReg * kReg];
    __shared__ int s_w[8];
    const int k = find_problem(A, blockIdx.x, false);
    const SweptProblem &p = A.prob[k];
    const Grid G = grid_of(A, p);
    const double *samp = A.samp + 3 * (int64_t)p.samp0;
    const int tile = (int)(blockIdx.x - p.tile0);
    const int tx = tile % p.tiles_x, ty = tile / p.tiles_x;
    const int a0 = tx * kSweptTile, b0 = ty * kSweptTile;
    // bounding box of the region's corners that lie in the grid
    const double bx0 = corner_x(G, max(a0 - 1, 0)), bx1 = corner_x(G, min(a0 + kSweptTile, G.nx - 1));
    const double by0 = corner_y(G, max(b0 - 1, 0)), by1 = corner_y(G, min(b0 + kSweptTile, G.ny - 1));
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    // a sample that reaches a corner of the region reaches its box: the rounded differences and squares are monotone, so the
    // box distance is never larger than the corner distance computed below
    for (int q = threadIdx.x; q < p.n_samp; q += blockDim.x) {
        const double sx = samp[3 * q], sy = samp[3 * q + 1], r = samp[3 * q + 2];
        const double dx = fmax(fmax(bx0 - sx, sx - bx1), 0.0), dy = fmax(fmax(by0 - sy, sy - by1), 0.0);
        if (dx * dx + dy * dy <= r * r) s_list[atomicAdd(&s_n, 1)] = q;
    }
    __syncthreads();
    const int n = s_n;
    for (int r = threadIdx.x; r < kReg * kReg; r += blockDim.x) {
        const int a = a0 - 1 + r % kReg, b = b0 - 1 + r / kReg;
        unsigned char u = 0;
        if (a >= 0 && a < G.nx && b >= 0 && b < G.ny) {
            const double px = corner_x(G, a), py = corner_y(G, b);
            for (int q = 0; q < n && !u; ++q) {
                const int s = s_list[q];
                const double sx = samp[3 * s], sy = samp[3 * s + 1], rr = samp[3 * s + 2];
                const double dx = px - sx, dy = py - sy;
                u = (dx * dx + dy * dy <= rr * rr) ? 1 : 0;
            }
        }
        s_unp[r] = u;
    }
    __syncthreads();
    const int la = threadIdx.x % kSweptTile, lb = threadIdx.x / kSweptTile;
    const int a = a0 + la, b = b0 + lb;
    int nd = 0;
    if (a < G.nx && b < G.ny) {
        // needed: one of the (up to four) cells around the corner has an unproven corner
        for (int cb = b - 1; cb <= b; ++cb)
            for (int ca = a - 1; ca <= a; ++ca) {
                if (ca < 0 || cb < 0 || ca > G.nx - 2 || cb > G.ny - 2) continue;
                const int ra = ca - a0 + 1, rb = cb - b0 + 1;
                nd |= s_unp[rb * kReg + ra] | s_unp[rb * kReg + ra + 1] | s_unp[(rb + 1) * kReg + ra] | s_unp[(rb + 1) * kReg + ra + 1];
            }
        const int64_t c = (int64_t)b * G.nx + a;
        G.need[c] = (unsigned char)nd;
        G.field[c] = __longlong_as_double(0x7ff8000000000000LL);
    }
    int total;
    block_scan256(nd, s_w, &total);
    if (threadIdx.x == 0) {
        A.tile_off[blockIdx.x] = total;
        if (total) atomicAdd(&A.stat[8 * k + 7], total);
    }
}

__global__ void __launch_bounds__(256) k_sw_compact(SweptArgs A) {
    __shared__ int s_w[8];
    const SweptProblem &p = A.prob[find_problem(A, blockIdx.x, false)];
    const Grid G = grid_of(A, p);
    const int tile = (int)(blockIdx.x - p.tile0);
    const int tx = tile % p.tiles_x, ty = tile / p.tiles_x;
    const int a = tx * kSweptTile + threadIdx.x % kSweptTile, b = ty * kSweptTile + threadIdx.x / kSweptTile;
    const bool in_grid = a < G.nx && b < G.ny;
    const int64_t c = (int64_t)b * G.nx + a;
    const int nd = in_grid ? G.need[c] : 0;
    int total;
    const int rank = block_scan256(nd, s_w, &total);
    if (nd) {
        const int64_t pos = (int64_t)A.tile_off[blockIdx.x] + rank;
        A.pts[2 * pos] = corner_x(G, a);
        A.pts[2 * pos + 1] = corner_y(G, b);
        A.idx[pos] = (int64_t)kSweptBlock * p.blk0 + c;
    }
}

__global__ void __launch_bounds__(256) k_sw_scatter(SweptArgs A) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= A.P) return;
    A.field[A.idx[k]] = A.val[k];
}

// ---- marching squares ---------------------------------------------------------------------------------------------------------
// Cell (a, b): corners c0 = (a, b), c1 = (a + 1, b), c2 = (a + 1, b + 1), c3 = (a, b + 1) (counter-clockwise); edges e0 = c0c1
// (horizontal edge of corner (a, b)), e1 = c1c2 (vertical edge of (a + 1, b)), e2 = c3c2 (horizontal edge of (a, b + 1)), e3 = c0c3
// (vertical edge of (a, b)).  Walk items 0..7 = c0, e0, c1, e1, c2, e2, c3, e3: corner k = item 2k, edge k = item 2k + 1.

struct CellPolys {
    int n;          // polygons: 0, 1 or 2
    int len[2];
    int item[2][6];
};

// The inside polygon(s) of a cell in walk order.  Separated saddles (m > iso): one triangle per inside corner with its two edges.
__device__ __forceinline__ void cell_polys(const bool in[4], bool connected, CellPolys &P) {
    bool have[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        have[2 * k] = in[k];
        have[2 * k + 1] = in[k] != in[(k + 1) & 3];
    }
    const int cas = (int)in[0] | ((int)in[1] << 1) | ((int)in[2] << 2) | ((int)in[3] << 3);
    P.n = 0;
    P.len[0] = P.len[1] = 0;
    if (cas == 0) return;
    if ((cas == 5 || cas == 10) && !connected) {
        P.n = 2;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (!in[k]) continue;
            const int p = k >> 1;  // corners 0, 2 (case 5) or 1, 3 (case 10): first and second polygon
            int l = 0;
#pragma unroll
            for (int it = 0; it < 8; ++it)
                if (it == 2 * k || it == 2 * k + 1 || it == ((2 * k + 7) & 7)) P.item[p][l++] = it;
            P.len[p] = l;
        }
        return;
    }
    P.n = 1;
    int l = 0;
#pragma unroll
    for (int it = 0; it < 8; ++it)
        if (have[it]) P.item[0][l++] = it;
    P.len[0] = l;
}

__device__ __forceinline__ int poly_segments(const CellPolys &P, int p) {
    int s = 0;
    for (int k = 0; k < P.len[p]; ++k) s += (P.item[p][k] & 1) && (P.item[p][(k + 1) % P.len[p]] & 1);
    return s;
}

struct CornerCounts {
    int h, v, c, s, f;   // crossing horizontal edge, crossing vertical edge, inside corner, segments and triangles of the cell
    int border_inside;
    int nonfinite;       // an evaluated corner with a non-finite value
};

__device__ __forceinline__ bool is_in(const Grid &G, int64_t c) { return G.field[c] <= G.iso; }  // NaN (not evaluated): outside

__device__ __forceinline__ bool cell_setup(const Grid &G, int a, int b, bool in[4], bool &connected) {
    if (a > G.nx - 2 || b > G.ny - 2) return false;
    const int64_t c = (int64_t)b * G.nx + a;
    if (!(G.need[c] && G.need[c + 1] && G.need[c + G.nx] && G.need[c + G.nx + 1])) return false;
    const double f00 = G.field[c], f10 = G.field[c + 1], f11 = G.field[c + G.nx + 1], f01 = G.field[c + G.nx];
    in[0] = f00 <= G.iso;
    in[1] = f10 <= G.iso;
    in[2] = f11 <= G.iso;
    in[3] = f01 <= G.iso;
    const double m = __dmul_rn(__dadd_rn(__dadd_rn(f00, f10), __dadd_rn(f01, f11)), 0.25);
    connected = m <= G.iso;
    return true;
}

__device__ __forceinline__ CornerCounts corner_counts(const Grid &G, int64_t c) {
    CornerCounts r{0, 0, 0, 0, 0, 0, 0};
    const int a = (int)(c % G.nx), b = (int)(c / G.nx);
    if (!G.need[c]) return r;
    r.nonfinite = !isfinite(G.field[c]);
    const bool ic = is_in(G, c);
    if (a < G.nx - 1 && G.need[c + 1]) r.h = ic != is_in(G, c + 1);
    if (b < G.ny - 1 && G.need[c + G.nx]) r.v = ic != is_in(G, c + G.nx);
    r.c = ic;
    r.border_inside = ic && (a == 0 || b == 0 || a == G.nx - 1 || b == G.ny - 1);
    bool in[4], conn;
    if (cell_setup(G, a, b, in, conn)) {
        CellPolys P;
        cell_polys(in, conn, P);
        for (int p = 0; p < P.n; ++p) {
            r.s += poly_segments(P, p);
            r.f += P.len[p] - 2;
        }
    }
    return r;
}

// The marching-squares CTA's problem and corners: block blockIdx.x is block lb of problem k, corners lb * kSweptBlock + 4 t + q.
struct BlockView {
    int k;
    const SweptProblem *p;
    Grid G;
    int64_t c0, n;  // first local corner of the CTA, corners of the problem
};
__device__ __forceinline__ BlockView block_view(const SweptArgs &A) {
    BlockView v;
    v.k = find_problem(A, blockIdx.x, true);
    v.p = &A.prob[v.k];
    v.G = grid_of(A, *v.p);
    v.c0 = (int64_t)(blockIdx.x - v.p->blk0) * kSweptBlock;
    v.n = (int64_t)v.G.nx * v.G.ny;
    return v;
}

__global__ void __launch_bounds__(256) k_sw_count(SweptArgs A) {
    __shared__ int s_w[5][8];
    const BlockView V = block_view(A);
    const int nblk = gridDim.x;
    int acc[5] = {0, 0, 0, 0, 0};
    int clip = 0, nonfinite = 0;
    for (int q = 0; q < 4; ++q) {
        const int64_t c = V.c0 + threadIdx.x * 4 + q;
        if (c >= V.n) break;
        const CornerCounts r = corner_counts(V.G, c);
        acc[0] += r.h; acc[1] += r.v; acc[2] += r.c; acc[3] += r.s; acc[4] += r.f;
        clip |= r.border_inside;
        nonfinite |= r.nonfinite;
    }
    int *st = A.stat + 8 * V.k;
    if (nonfinite) atomicOr(&st[0], 1);
    if (clip) atomicOr(&st[1], 1);
#pragma unroll
    for (int ch = 0; ch < 5; ++ch) {
        int total;
        block_scan256(acc[ch], s_w[ch], &total);
        if (threadIdx.x == 0) {
            A.blk[ch * (nblk + 1) + blockIdx.x] = total;
            if (total) atomicAdd(&st[2 + ch], total);
        }
    }
}

__global__ void __launch_bounds__(256) k_sw_vertices(SweptArgs A) {
    __shared__ int s_w[3][8];
    const BlockView V = block_view(A);
    const int nblk = gridDim.x;
    const int64_t b0 = V.p->blk0, b1 = b0 + V.p->nblk;
    CornerCounts r[4];
    int acc[3] = {0, 0, 0};
    for (int q = 0; q < 4; ++q) {
        const int64_t c = V.c0 + threadIdx.x * 4 + q;
        r[q] = (c < V.n) ? corner_counts(V.G, c) : CornerCounts{0, 0, 0, 0, 0, 0, 0};
        acc[0] += r[q].h; acc[1] += r[q].v; acc[2] += r[q].c;
    }
    // the problem's vertices: horizontal-edge, vertical-edge, then corner vertices, from its first vertex `vbase` of the concatenation
    int base[3], tot[3];
    int64_t vbase = 0;
    for (int ch = 0; ch < 3; ++ch) {
        const int *row = A.blk + ch * (nblk + 1);
        int total;
        base[ch] = block_scan256(acc[ch], s_w[ch], &total) + row[blockIdx.x] - row[b0];
        tot[ch] = row[b1] - row[b0];
        vbase += row[b0];
    }
    base[1] += tot[0];
    base[2] += tot[0] + tot[1];
    double *verts = A.verts + 2 * vbase;
    for (int q = 0; q < 4; ++q) {
        const int64_t c = V.c0 + threadIdx.x * 4 + q;
        if (c >= V.n) break;
        const int64_t a = c % V.G.nx, b = c / V.G.nx;
        const double x = corner_x(V.G, a), y = corner_y(V.G, b);
        int *vid = V.G.vid + 3 * c;
        if (r[q].h) {  // edge (a, b) - (a + 1, b)
            const double fa = V.G.field[c], fb = V.G.field[c + 1];
            const double s = __ddiv_rn(__dsub_rn(A.iso, fa), __dsub_rn(fb, fa));
            const double xb = corner_x(V.G, a + 1);
            const int id = base[0]++;
            verts[2 * (int64_t)id] = __dadd_rn(x, __dmul_rn(s, __dsub_rn(xb, x)));
            verts[2 * (int64_t)id + 1] = __dadd_rn(y, __dmul_rn(s, __dsub_rn(y, y)));
            vid[0] = id;
        }
        if (r[q].v) {  // edge (a, b) - (a, b + 1)
            const double fa = V.G.field[c], fb = V.G.field[c + V.G.nx];
            const double s = __ddiv_rn(__dsub_rn(A.iso, fa), __dsub_rn(fb, fa));
            const double yb = corner_y(V.G, b + 1);
            const int id = base[1]++;
            verts[2 * (int64_t)id] = __dadd_rn(x, __dmul_rn(s, __dsub_rn(x, x)));
            verts[2 * (int64_t)id + 1] = __dadd_rn(y, __dmul_rn(s, __dsub_rn(yb, y)));
            vid[1] = id;
        }
        if (r[q].c) {
            const int id = base[2]++;
            verts[2 * (int64_t)id] = x;
            verts[2 * (int64_t)id + 1] = y;
            vid[2] = id;
        }
    }
}

__global__ void __launch_bounds__(256) k_sw_cells(SweptArgs A) {
    __shared__ int s_w[2][8];
    const BlockView V = block_view(A);
    const int nblk = gridDim.x;
    int acc[2] = {0, 0};
    for (int q = 0; q < 4; ++q) {
        const int64_t c = V.c0 + threadIdx.x * 4 + q;
        if (c >= V.n) break;
        const CornerCounts r = corner_counts(V.G, c);
        acc[0] += r.s; acc[1] += r.f;
    }
    // segment and triangle positions in the concatenation (problem by problem); the vertex ids they hold are the problem's own
    int total;
    int64_t so = block_scan256(acc[0], s_w[0], &total) + (int64_t)A.blk[3 * (nblk + 1) + blockIdx.x];
    int64_t fo = block_scan256(acc[1], s_w[1], &total) + (int64_t)A.blk[4 * (nblk + 1) + blockIdx.x];
    const Grid &G = V.G;
    for (int q = 0; q < 4; ++q) {
        const int64_t c = V.c0 + threadIdx.x * 4 + q;
        if (c >= V.n) break;
        bool in[4], conn;
        if (!cell_setup(G, (int)(c % G.nx), (int)(c / G.nx), in, conn)) continue;
        CellPolys P;
        cell_polys(in, conn, P);
        if (P.n == 0) continue;
        const int64_t nx = G.nx;
        // vertex of every walk item
        const int id[8] = {G.vid[3 * c + 2], G.vid[3 * c + 0], G.vid[3 * (c + 1) + 2], G.vid[3 * (c + 1) + 1],
                           G.vid[3 * (c + nx + 1) + 2], G.vid[3 * (c + nx) + 0], G.vid[3 * (c + nx) + 2], G.vid[3 * c + 1]};
        for (int p = 0; p < P.n; ++p) {
            const int L = P.len[p];
            for (int k = 0; k < L; ++k) {
                const int u = P.item[p][k], w = P.item[p][(k + 1) % L];
                if ((u & 1) && (w & 1)) {
                    A.segs[2 * so] = id[u];
                    A.segs[2 * so + 1] = id[w];
                    ++so;
                }
            }
            for (int k = 1; k + 1 < L; ++k) {
                A.tris[3 * fo] = id[P.item[p][0]];
                A.tris[3 * fo + 1] = id[P.item[p][k]];
                A.tris[3 * fo + 2] = id[P.item[p][k + 1]];
                ++fo;
            }
        }
    }
}

// exclusive prefix of `channels` rows of n counts (row stride n + 1; the row's total lands at [n] and at totals[ch])
__global__ void __launch_bounds__(1024) k_sw_scan(int *counts, int n, int channels, int *totals) {
    __shared__ int s_w[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int ch = 0; ch < channels; ++ch) {
        int *row = counts + (int64_t)ch * (n + 1);
        int carry = 0;
        for (int base = 0; base < n; base += 1024) {
            const int i = base + threadIdx.x;
            const int v = (i < n) ? row[i] : 0;
            int x = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, x, o);
                if (lane >= o) x += y;
            }
            if (lane == 31) s_w[warp] = x;
            __syncthreads();
            int before = 0, all = 0;
            for (int w = 0; w < 32; ++w) {
                const int s = s_w[w];
                if (w < warp) before += s;
                all += s;
            }
            __syncthreads();
            if (i < n) row[i] = carry + before + x - v;
            carry += all;
        }
        if (threadIdx.x == 0) row[n] = totals[ch] = carry;
        __syncthreads();
    }
}

}  // namespace

cudaError_t launch_swept(int what, const SweptArgs &A, cudaStream_t st) {
    switch (what) {
        case 0: k_sw_classify<<<A.tiles, 256, 0, st>>>(A); break;
        case 1: k_sw_compact<<<A.tiles, 256, 0, st>>>(A); break;
        case 2: k_sw_scatter<<<(unsigned)((A.P + 255) / 256), 256, 0, st>>>(A); break;
        case 3: k_sw_count<<<A.n_blocks, 256, 0, st>>>(A); break;
        case 4: k_sw_vertices<<<A.n_blocks, 256, 0, st>>>(A); break;
        case 5: k_sw_cells<<<A.n_blocks, 256, 0, st>>>(A); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

cudaError_t launch_swept_scan(int *counts, int n, int channels, int *totals, cudaStream_t st) {
    k_sw_scan<<<1, 1024, 0, st>>>(counts, n, channels, totals);
    return cudaGetLastError();
}

}  // namespace svsdf
