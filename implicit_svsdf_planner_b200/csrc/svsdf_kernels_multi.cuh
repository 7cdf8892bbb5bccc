// svsdf_kernels_multi.cuh — svsdf_cost_grad_multi: the cost and gradient of n problems (each its own trajectory and query points, one
// robot) in one set of launches: k_pose_table_multi, k_outer_multi (one launch per schedule that occurs), k_compact_multi,
// k_gsip_multi, k_finalize_multi.  The kernels run the single-problem bodies of svsdf_kernels.cuh on a per-problem view chosen at the
// top of the CTA (or of the inside slot), so every problem gets the bits svsdf_cost_grad gives it:
//  * k_outer_multi: physical CTA c is virtual CTA v of problem k (MultiArgs::cta_map); outer_body runs with vblock = v and
//    vgrid = the problem's own grid, and writes the problem's partials [grid][19N + 1].
//  * k_compact_multi: one CTA per problem (ascending inside list per problem); the last CTA turns the counts into slot offsets.
//  * k_gsip_multi: one queue over the concatenated inside lists; slot s belongs to the problem k with ins_off[k] <= s < ins_off[k + 1].
//  * k_finalize_multi: blockIdx.y = problem; k_finalize's fixed tree over the problem's grid, then its inside contributions in
//    ascending point order.
// Included by svsdf_kernels_multi_{fast,strict}.cu (rigid; these also carry the pose / compaction / finalize kernels) and
// svsdf_kernels_multi_scaled_{fast,strict}.cu (SVSDF_SCALED_UNIT: the deformable-robot k_outer_multi / k_gsip_multi), after
// svsdf_kernels.cuh with SVSDF_MULTI_UNIT defined.
#pragma once
#include "svsdf_kernels.cuh"

namespace svsdf {
namespace SVSDF_NS {

template <int SHAPE, bool XFORM, bool BATCHED, bool SCALED>
__device__ __forceinline__ void outer_multi_body(const KernelArgs &A, const MultiArgs &M, const ShapeParams &S, const ScaleSched *Z) {
    const int k = M.cta_map[2 * blockIdx.x], v = M.cta_map[2 * blockIdx.x + 1];
    const MultiProblem pr = M.prob[k];
    KernelArgs Ak = A;
    Ak.blob = A.blob + pr.blob_off;
    Ak.blob_doubles = pr.blob_doubles;
    Ak.points_xy = A.points_xy + 2 * pr.pt_off;
    Ak.P = pr.P;
    Ak.partials = A.partials + pr.part_off;
    Ak.inside_flag = A.inside_flag + pr.flag_off;
    Ak.inside_tstar = A.inside_tstar + pr.pt_off;
    outer_body<SHAPE, XFORM, BATCHED, SCALED>(Ak, S, Z, v, pr.grid);
}
template <int SHAPE, bool XFORM, bool BATCHED>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, (SHAPE == SH_MESH) ? SVSDF_MESH_MIN_CTAS : SVSDF_OUTER_MIN_CTAS)
    k_outer_multi(const __grid_constant__ KernelArgs A, const __grid_constant__ MultiArgs M, const __grid_constant__ ShapeParams S) {
    outer_multi_body<SHAPE, XFORM, BATCHED, false>(A, M, S, nullptr);
}
template <int SHAPE, bool XFORM, bool BATCHED>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, (SHAPE == SH_MESH) ? SVSDF_MESH_MIN_CTAS : SVSDF_OUTER_MIN_CTAS)
    k_outer_multi_scaled(const __grid_constant__ KernelArgs A, const __grid_constant__ MultiArgs M, const __grid_constant__ ShapeParams S,
                         const __grid_constant__ ScaleSched Z) {
    outer_multi_body<SHAPE, XFORM, BATCHED, true>(A, M, S, &Z);
}

// Reload of the CTA's blob buffer for the next problem: the barrier was initialised by tma_load_blob and has completed `parity`
// phases' worth of loads; every thread has left the previous wait and finished reading the old blob (__syncthreads before the call).
__device__ __forceinline__ void tma_reload_blob(double *smem_blob, const double *gmem_blob, int n_doubles, uint64_t *bar, uint32_t parity) {
    const uint32_t bar_a = smem_u32(bar);
    const uint32_t bytes = (uint32_t)n_doubles * 8u;
    if (threadIdx.x == 0) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the generic-proxy reads of the old blob come first
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_blob)),
            "l"(gmem_blob), "r"(bytes), "r"(bar_a)
            : "memory");
    }
    uint32_t done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar_a), "r"(parity)
            : "memory");
    }
}

// k_gsip_multi's view of the inside slots (gsip_body): slot s of the concatenated lists belongs to the last problem k with
// ins_off[k] <= s (problems without inside points are skipped); the CTA's blob is reloaded when the problem changes.
struct GsipMulti {
    const KernelArgs &A;
    const MultiArgs &M;
    int *loaded;      // problem whose blob is in shared memory (-1: none yet)
    uint32_t *phase;  // mbarrier phase of the next load
    __device__ __forceinline__ void start(double *, uint64_t *) const {}
    __device__ __forceinline__ int count() const { return M.ins_off[M.n]; }
    __device__ __forceinline__ bool at(int slot, double *sblob, uint64_t *bar, int &pt, const double *&pts, const double *&tstar) const {
        int lo = 0, hi = M.n - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (M.ins_off[mid] <= slot) lo = mid;
            else hi = mid - 1;
        }
        const MultiProblem &pr = M.prob[lo];
        pt = A.inside_list[pr.pt_off + (slot - M.ins_off[lo])];
        pts = A.points_xy + 2 * pr.pt_off;
        tstar = A.inside_tstar + pr.pt_off;
        if (lo == *loaded) return false;
        if (*loaded < 0) {
            tma_load_blob(sblob, A.blob + pr.blob_off, pr.blob_doubles, bar);
        } else {
            __syncthreads();  // every thread is done with the previous blob
            tma_reload_blob(sblob, A.blob + pr.blob_off, pr.blob_doubles, bar, *phase);
        }
        *phase ^= 1u;
        *loaded = lo;
        return true;
    }
};
template <int SHAPE, bool XFORM, int WARPS, bool SCALED>
__device__ __forceinline__ void gsip_multi_body(const KernelArgs &A, const MultiArgs &M, const ShapeParams &S, const ScaleSched *Z) {
    int loaded = -1;
    uint32_t phase = 0;
    gsip_body<SHAPE, XFORM, WARPS, SCALED>(A, S, Z, GsipMulti{A, M, &loaded, &phase});
}
template <int SHAPE, bool XFORM, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, (WARPS == kWarpsPerBlock && SHAPE != SH_MESH) ? SVSDF_GSIP_MIN_CTAS : 1)
    k_gsip_multi(const __grid_constant__ KernelArgs A, const __grid_constant__ MultiArgs M, const __grid_constant__ ShapeParams S) {
    gsip_multi_body<SHAPE, XFORM, WARPS, false>(A, M, S, nullptr);
}
template <int SHAPE, bool XFORM, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, (WARPS == kWarpsPerBlock && SHAPE != SH_MESH) ? SVSDF_GSIP_MIN_CTAS : 1)
    k_gsip_multi_scaled(const __grid_constant__ KernelArgs A, const __grid_constant__ MultiArgs M, const __grid_constant__ ShapeParams S,
                        const __grid_constant__ ScaleSched Z) {
    gsip_multi_body<SHAPE, XFORM, WARPS, true>(A, M, S, &Z);
}

#ifndef SVSDF_SCALED_UNIT
// grid (ceil(max K1 / 128), n): one thread per (problem, layer-1 sample)
__global__ void k_pose_table_multi(double *blobs, const __grid_constant__ MultiArgs M) {
    const MultiProblem pr = M.prob[blockIdx.y];
    pose_table_entry(blobs + pr.blob_off, blockIdx.x * blockDim.x + threadIdx.x);
}

// one CTA per problem; the last CTA to finish writes the slot offsets of the concatenated inside lists
__global__ void __launch_bounds__(1024) k_compact_multi(const unsigned char *flag, int *list, const __grid_constant__ MultiArgs M) {
    const MultiProblem pr = M.prob[blockIdx.x];
    compact_body(flag + pr.flag_off, pr.P, list + pr.pt_off, M.ins_count + blockIdx.x);
    __shared__ bool last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = (atomicAdd(M.compact_ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!last) return;
    __threadfence();
    if (threadIdx.x == 0) {  // n is at most a few thousand: a serial scan is a few microseconds
        int s = 0;
        for (int k = 0; k < M.n; ++k) {
            M.ins_off[k] = s;
            s += __ldcg(M.ins_count + k);
        }
        M.ins_off[M.n] = s;
        *M.compact_ticket = 0u;
    }
}

// grid (ceil(max(19N + 1) / 8), n): problem k uses the first ceil((19 N_k + 1) / 8) CTAs of its row
__global__ void __launch_bounds__(256) k_finalize_multi(const double *partials, const double *gsip_contrib, const int *gsip_piece,
                                                        const __grid_constant__ MultiArgs M) {
    const int k = blockIdx.y;
    const MultiProblem pr = M.prob[k];
    const int nbx = (19 * pr.N + 1 + 7) / 8;
    if ((int)blockIdx.x >= nbx) return;
    const int off = M.ins_off[k];
    finalize_body(partials + pr.part_off, pr.grid, pr.N, M.ins_off[k + 1] - off, gsip_contrib + 20 * (int64_t)off, gsip_piece + off,
                  M.tot + pr.out_off, M.tickets + k, M.out + pr.out_off, blockIdx.x, nbx);
}
#endif

// ---- launchers ------------------------------------------------------------------------------------------------------------------
template <int SHAPE, bool XFORM>
static cudaError_t multi_attrs() {
    static bool attr_set_dev[64] = {};
    int dev_ord = 0;
    cudaGetDevice(&dev_ord);
    bool &attr_set = attr_set_dev[dev_ord & 63];
    if (attr_set) return cudaSuccess;
    const void *k[4];
    if constexpr (kScaledUnit) {
        k[0] = (const void *)k_outer_multi_scaled<SHAPE, XFORM, false>;
        k[1] = (const void *)k_outer_multi_scaled<SHAPE, XFORM, true>;
        k[2] = (const void *)k_gsip_multi_scaled<SHAPE, XFORM, kWarpsPerBlock>;
        k[3] = (const void *)k_gsip_multi_scaled<SHAPE, XFORM, kGsipWarps>;
    } else {
        k[0] = (const void *)k_outer_multi<SHAPE, XFORM, false>;
        k[1] = (const void *)k_outer_multi<SHAPE, XFORM, true>;
        k[2] = (const void *)k_gsip_multi<SHAPE, XFORM, kWarpsPerBlock>;
        k[3] = (const void *)k_gsip_multi<SHAPE, XFORM, kGsipWarps>;
    }
    for (int i = 0; i < 4; ++i) {
        cudaError_t e = cudaFuncSetAttribute(k[i], cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        if (e != cudaSuccess) return e;
    }
    attr_set = true;
    return cudaSuccess;
}

// what: 0 sparse k_outer_multi, 1 batched k_outer_multi, 2 k_gsip_multi (gsip_wide: the 22-warp variant; grid <= 0: resident
// CTAs per SM x SMs of the chosen variant)
template <int SHAPE, bool XFORM>
static cudaError_t launch_multi_shape(int what, const KernelArgs &A, const MultiArgs &M, const ShapeParams &S, const ScaleSched *Z,
                                      int grid, size_t smem, int gsip_wide, int sm_count, cudaStream_t st) {
    cudaError_t e = multi_attrs<SHAPE, XFORM>();
    if (e != cudaSuccess) return e;
    constexpr int TO = kWarpsPerBlock * 32;
    if (what == 0 || what == 1) {
        if constexpr (kScaledUnit) {
            if (what == 1) k_outer_multi_scaled<SHAPE, XFORM, true><<<grid, TO, smem, st>>>(A, M, S, *Z);
            else k_outer_multi_scaled<SHAPE, XFORM, false><<<grid, TO, smem, st>>>(A, M, S, *Z);
        } else {
            if (what == 1) k_outer_multi<SHAPE, XFORM, true><<<grid, TO, smem, st>>>(A, M, S);
            else k_outer_multi<SHAPE, XFORM, false><<<grid, TO, smem, st>>>(A, M, S);
        }
        return cudaGetLastError();
    }
    const void *kg;
    if constexpr (kScaledUnit) kg = gsip_wide ? (const void *)k_gsip_multi_scaled<SHAPE, XFORM, kGsipWarps> : (const void *)k_gsip_multi_scaled<SHAPE, XFORM, kWarpsPerBlock>;
    else kg = gsip_wide ? (const void *)k_gsip_multi<SHAPE, XFORM, kGsipWarps> : (const void *)k_gsip_multi<SHAPE, XFORM, kWarpsPerBlock>;
    const int threads = gsip_wide ? kGsipWarps * 32 : TO;
    if (grid <= 0) {
        int occ = 0;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kg, threads, smem);
        if (e != cudaSuccess) return e;
        grid = gsip_wide ? sm_count : sm_count * (occ > 0 ? occ : 1);
    }
    if constexpr (kScaledUnit) {
        if (gsip_wide) k_gsip_multi_scaled<SHAPE, XFORM, kGsipWarps><<<grid, threads, smem, st>>>(A, M, S, *Z);
        else k_gsip_multi_scaled<SHAPE, XFORM, kWarpsPerBlock><<<grid, threads, smem, st>>>(A, M, S, *Z);
    } else {
        if (gsip_wide) k_gsip_multi<SHAPE, XFORM, kGsipWarps><<<grid, threads, smem, st>>>(A, M, S);
        else k_gsip_multi<SHAPE, XFORM, kWarpsPerBlock><<<grid, threads, smem, st>>>(A, M, S);
    }
    return cudaGetLastError();
}

cudaError_t launch_multi(int what, const KernelArgs &A, const MultiArgs &M, const ShapeParams &S, const ScaleSched *Z, int grid, size_t smem,
                         int gsip_wide, int sm_count, cudaStream_t st) {
    const bool xf = S.has_xform != 0;
    switch (S.id) {
#define SVSDF_CASE(ID)                                                                                      \
    case ID:                                                                                                \
        return xf ? launch_multi_shape<ID, true>(what, A, M, S, Z, grid, smem, gsip_wide, sm_count, st)     \
                  : launch_multi_shape<ID, false>(what, A, M, S, Z, grid, smem, gsip_wide, sm_count, st);
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
        case SH_POLYGON: return launch_multi_shape<SH_POLYGON, false>(what, A, M, S, Z, grid, smem, gsip_wide, sm_count, st);
        case SH_MESH: return launch_multi_shape<SH_MESH, false>(what, A, M, S, Z, grid, smem, gsip_wide, sm_count, st);
        default: return cudaErrorInvalidValue;
    }
}

#ifndef SVSDF_SCALED_UNIT
cudaError_t launch_pose_multi(double *blobs, const MultiArgs &M, int max_K1, cudaStream_t st) {
    k_pose_table_multi<<<dim3((max_K1 + 127) / 128, M.n), 128, 0, st>>>(blobs, M);
    return cudaGetLastError();
}
cudaError_t launch_compact_multi(const unsigned char *flag, int *list, const MultiArgs &M, cudaStream_t st) {
    k_compact_multi<<<M.n, 1024, 0, st>>>(flag, list, M);
    return cudaGetLastError();
}
cudaError_t launch_finalize_multi(const double *partials, const double *gsip_contrib, const int *gsip_piece, const MultiArgs &M, int max_N,
                                  cudaStream_t st) {
    k_finalize_multi<<<dim3((19 * max_N + 1 + 7) / 8, M.n), 256, 0, st>>>(partials, gsip_contrib, gsip_piece, M);
    return cudaGetLastError();
}
#endif

}  // namespace SVSDF_NS
}  // namespace svsdf
