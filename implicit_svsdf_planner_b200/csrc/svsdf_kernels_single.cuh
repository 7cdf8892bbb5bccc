// svsdf_kernels_single.cuh — the single-problem cost launchers (svsdf_cost_grad and the point queries): k_outer, k_compact, k_gsip.
// Included by svsdf_kernels{,_scaled}_{fast,strict}.cu; SVSDF_SCALED (0 / 1) selects the rigid or the deformable-robot kernels.
#pragma once
#include "svsdf_kernels.cuh"

namespace svsdf {
namespace SVSDF_NS {

__global__ void __launch_bounds__(1024) k_compact(const unsigned char *flag, int64_t P, int *list, int *n_out) {
    compact_body(flag, P, list, n_out);
}

// the cost kernels of a single-problem variant, as raise_smem_cap and launch_cost take them
template <int SHAPE, bool XFORM, bool SCALED>
struct CostKernels {
    static auto outer(bool batched) { return batched ? k_outer<SHAPE, XFORM, true> : k_outer<SHAPE, XFORM, false>; }
    static auto gsip(bool wide) { return wide ? k_gsip<SHAPE, XFORM, kGsipWarps> : k_gsip<SHAPE, XFORM, kWarpsPerBlock>; }
};
template <int SHAPE, bool XFORM>
struct CostKernels<SHAPE, XFORM, true> {
    static auto outer(bool batched) { return batched ? k_outer_scaled<SHAPE, XFORM, true> : k_outer_scaled<SHAPE, XFORM, false>; }
    static auto gsip(bool wide) { return wide ? k_gsip_scaled<SHAPE, XFORM, kGsipWarps> : k_gsip_scaled<SHAPE, XFORM, kWarpsPerBlock>; }
};

struct LaunchCfg {
    int grid_outer, grid_gsip;
    size_t smem_outer, smem_gsip;
    cudaStream_t stream;
    cudaEvent_t after_outer;  // optional timing mark recorded right after k_outer
    bool gsip_wide;           // use the 22-warp k_gsip variant
};

template <int SHAPE, bool XFORM>
static cudaError_t launch_shape(const KernelArgs &A, const ShapeParams &S, const ScaleSched *Z, const LaunchCfg &cfg) {
    using K = CostKernels<SHAPE, XFORM, SVSDF_SCALED>;
    cudaError_t e = raise_smem_cap<K>();
    if (e != cudaSuccess) return e;
    e = launch_cost<SVSDF_SCALED>(K::outer(A.batched), cfg.grid_outer, kWarpsPerBlock * 32, cfg.smem_outer, cfg.stream, Z, A, S);
    if (e != cudaSuccess) return e;
    if (cfg.after_outer) cudaEventRecord(cfg.after_outer, cfg.stream);
    if (A.want_gsip) {
        k_compact<<<1, 1024, 0, cfg.stream>>>(A.inside_flag, A.P, A.inside_list, A.n_inside);
        // few inside points: one warp per ring sample (latency); many: 8-warp CTAs, two per SM (throughput)
        const int threads = (cfg.gsip_wide ? kGsipWarps : kWarpsPerBlock) * 32;
        e = launch_cost<SVSDF_SCALED>(K::gsip(cfg.gsip_wide), cfg.grid_gsip, threads, cfg.smem_gsip, cfg.stream, Z, A, S);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

template <int SHAPE, bool XFORM>
static cudaError_t occ_shape(int N, int blob_doubles, int *occ_outer, int *occ_gsip, int *chunk_outer) {
    const size_t smem_outer = outer_smem_doubles(blob_doubles, N, 1) * sizeof(double), smem_gsip = (size_t)blob_doubles * sizeof(double);
    using K = CostKernels<SHAPE, XFORM, SVSDF_SCALED>;
    cudaError_t e = raise_smem_cap<K>();
    if (e != cudaSuccess) return e;
    // the two schedules are compiled to the same register cap (launch bounds); the batched kernel sizes the full wave
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ_outer, K::outer(true), kWarpsPerBlock * 32, smem_outer);
    if (e != cudaSuccess) return e;
    // the largest chunk whose work area fits and leaves that residency alone (the grid is sized from it)
    for (*chunk_outer = kOuterChunkMax; *chunk_outer > 1; --*chunk_outer) {
        const size_t sc = outer_smem_doubles(blob_doubles, N, *chunk_outer) * sizeof(double);
        int occ = 0;
        if (sc > kMaxDynSmemBytes) continue;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, K::outer(true), kWarpsPerBlock * 32, sc);
        if (e != cudaSuccess) return e;
        if (occ == *occ_outer) break;
    }
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ_gsip, K::gsip(false), kWarpsPerBlock * 32, smem_gsip);
}

// Resident CTAs per SM of k_outer / k_gsip for this shape and trajectory size: the host sizes the grids as
// SMs x occupancy so that the warp-stride loops run as exactly one full wave (no partial second wave).  k_outer's is taken with a
// chunk of 1; *chunk_outer is the largest chunk (<= kOuterChunkMax) at which it is still the same.
cudaError_t query_occupancy(const ShapeParams &S, int N, int blob_doubles, int *occ_outer, int *occ_gsip, int *chunk_outer) {
    return dispatch_shape<ShapeSet::all>(
        S, [&](auto id, auto xf) { return occ_shape<id.value, xf.value>(N, blob_doubles, occ_outer, occ_gsip, chunk_outer); });
}

cudaError_t launch_cost_kernels(const KernelArgs &A, const ShapeParams &S, const ScaleSched *Z, int N, int grid_outer, int grid_gsip,
                                cudaStream_t stream, cudaEvent_t after_outer, int gsip_wide) {
    LaunchCfg cfg;
    cfg.after_outer = after_outer;
    cfg.gsip_wide = gsip_wide != 0;
    cfg.grid_outer = grid_outer;
    cfg.grid_gsip = grid_gsip;
    cfg.smem_outer = outer_smem_doubles(A.blob_doubles, N, A.batched ? A.outer_chunk : 1) * sizeof(double);
    cfg.smem_gsip = (size_t)A.blob_doubles * sizeof(double);
    cfg.stream = stream;
    return dispatch_shape<ShapeSet::all>(S, [&](auto id, auto xf) { return launch_shape<id.value, xf.value>(A, S, Z, cfg); });
}

}  // namespace SVSDF_NS
}  // namespace svsdf
