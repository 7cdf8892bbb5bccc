// svsdf_kernels_multi_shared.cuh — the multi-problem kernels every variant shares, so only the rigid multi units carry them
// (svsdf_kernels_multi_{fast,strict}.cu): k_pose_table_multi, k_compact_multi and k_finalize_multi, and their launchers.
#pragma once
#include "svsdf_kernels.cuh"

namespace svsdf {
namespace SVSDF_NS {

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

}  // namespace SVSDF_NS
}  // namespace svsdf
