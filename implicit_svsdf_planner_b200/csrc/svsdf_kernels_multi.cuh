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
// Included by svsdf_kernels_multi_{fast,strict}.cu (rigid; these also carry the pose / compaction / finalize kernels of
// svsdf_kernels_multi_shared.cuh) and svsdf_kernels_multi_scaled_{fast,strict}.cu; SVSDF_SCALED (0 / 1) selects the rigid or the
// deformable-robot k_outer_multi / k_gsip_multi.
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
    if (A.out_sdf) Ak.out_sdf = A.out_sdf + pr.pt_off;  // per-point outputs (svsdf_map_clearance_multi; null on the cost path)
    if (A.out_tstar) Ak.out_tstar = A.out_tstar + pr.pt_off;
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
// ins_off[k] <= s (problems without inside points are skipped); the CTA's blob is reloaded when the problem changes.  The point index
// it hands out counts from the start of the concatenated points (pt_off + the problem's own index), so the per-point outputs land at
// the point's place in the concatenation.
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
        pt = (int)pr.pt_off + A.inside_list[pr.pt_off + (slot - M.ins_off[lo])];
        pts = A.points_xy;
        tstar = A.inside_tstar;
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

// ---- launchers ------------------------------------------------------------------------------------------------------------------
// the cost kernels of a multi-problem variant, as raise_smem_cap and launch_cost take them
template <int SHAPE, bool XFORM, bool SCALED>
struct MultiKernels {
    static auto outer(bool batched) { return batched ? k_outer_multi<SHAPE, XFORM, true> : k_outer_multi<SHAPE, XFORM, false>; }
    static auto gsip(bool wide) { return wide ? k_gsip_multi<SHAPE, XFORM, kGsipWarps> : k_gsip_multi<SHAPE, XFORM, kWarpsPerBlock>; }
};
template <int SHAPE, bool XFORM>
struct MultiKernels<SHAPE, XFORM, true> {
    static auto outer(bool batched) { return batched ? k_outer_multi_scaled<SHAPE, XFORM, true> : k_outer_multi_scaled<SHAPE, XFORM, false>; }
    static auto gsip(bool wide) {
        return wide ? k_gsip_multi_scaled<SHAPE, XFORM, kGsipWarps> : k_gsip_multi_scaled<SHAPE, XFORM, kWarpsPerBlock>;
    }
};

// what: 0 sparse k_outer_multi, 1 batched k_outer_multi, 2 k_gsip_multi (gsip_wide: the 22-warp variant; grid <= 0: resident
// CTAs per SM x SMs of the chosen variant)
template <int SHAPE, bool XFORM>
static cudaError_t launch_multi_shape(int what, const KernelArgs &A, const MultiArgs &M, const ShapeParams &S, const ScaleSched *Z,
                                      int grid, size_t smem, int gsip_wide, int sm_count, cudaStream_t st) {
    using K = MultiKernels<SHAPE, XFORM, SVSDF_SCALED>;
    cudaError_t e = raise_smem_cap<K>();
    if (e != cudaSuccess) return e;
    if (what == 0 || what == 1) return launch_cost<SVSDF_SCALED>(K::outer(what == 1), grid, kWarpsPerBlock * 32, smem, st, Z, A, M, S);
    const auto kg = K::gsip(gsip_wide);
    const int threads = (gsip_wide ? kGsipWarps : kWarpsPerBlock) * 32;
    if (grid <= 0) {
        int occ = 0;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kg, threads, smem);
        if (e != cudaSuccess) return e;
        grid = gsip_wide ? sm_count : sm_count * (occ > 0 ? occ : 1);
    }
    return launch_cost<SVSDF_SCALED>(kg, grid, threads, smem, st, Z, A, M, S);
}

cudaError_t launch_multi(int what, const KernelArgs &A, const MultiArgs &M, const ShapeParams &S, const ScaleSched *Z, int grid, size_t smem,
                         int gsip_wide, int sm_count, cudaStream_t st) {
    return dispatch_shape<ShapeSet::all>(S, [&](auto id, auto xf) {
        return launch_multi_shape<id.value, xf.value>(what, A, M, S, Z, grid, smem, gsip_wide, sm_count, st);
    });
}

}  // namespace SVSDF_NS
}  // namespace svsdf
