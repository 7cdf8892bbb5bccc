// svsdf_launch.h — host-callable launchers exported by the two kernel translation units
// (svsdf_kernels_fast.cu: FMA contraction on; svsdf_kernels_strict.cu: -fmad=false).
#pragma once
#include <cuda_runtime.h>

#include "svsdf_types.h"

namespace svsdf {
#define SVSDF_DECLARE_LAUNCHERS(NS)                                                                              \
    namespace NS {                                                                                               \
    cudaError_t launch_pose_table(double *blob, int K1, cudaStream_t stream);                                    \
    cudaError_t query_occupancy(const ShapeParams &S, int N, int blob_doubles, int *occ_outer, int *occ_gsip);   \
    cudaError_t launch_cost_kernels(const KernelArgs &A, const ShapeParams &S, int N, int grid_outer,            \
                                    int grid_gsip, cudaStream_t stream, cudaEvent_t after_outer,                 \
                                    int gsip_wide);                                                              \
    cudaError_t launch_finalize(const double *partials, int n_blocks, int N, const int *n_inside,                \
                                const double *gsip_contrib, const int *gsip_piece, double *tot,                  \
                                unsigned int *ticket, double *out, cudaStream_t stream);                         \
    cudaError_t launch_shape_eval(const ShapeParams &S, const double *rel_xy, int64_t n, double *out, int grad,  \
                                  cudaStream_t stream);                                                          \
    cudaError_t launch_fp64_peak(double *out, int grid, int iters, cudaStream_t stream);                         \
    cudaError_t launch_sincos(const double *x, int64_t n, double *s, double *c, cudaStream_t stream);            \
    }
SVSDF_DECLARE_LAUNCHERS(fast)
SVSDF_DECLARE_LAUNCHERS(strict)
#undef SVSDF_DECLARE_LAUNCHERS
// deformable robots (svsdf_kernels_scaled_fast.cu / svsdf_kernels_scaled_strict.cu): the same cost kernels with the
// schedule Z as an extra kernel parameter
#define SVSDF_DECLARE_SCALED_LAUNCHERS(NS)                                                                       \
    namespace NS {                                                                                               \
    cudaError_t query_occupancy(const ShapeParams &S, int N, int blob_doubles, int *occ_outer, int *occ_gsip);   \
    cudaError_t launch_cost_kernels(const KernelArgs &A, const ShapeParams &S, const ScaleSched &Z, int N,       \
                                    int grid_outer, int grid_gsip, cudaStream_t stream, cudaEvent_t after_outer, \
                                    int gsip_wide);                                                              \
    }
SVSDF_DECLARE_SCALED_LAUNCHERS(fast_scaled)
SVSDF_DECLARE_SCALED_LAUNCHERS(strict_scaled)
#undef SVSDF_DECLARE_SCALED_LAUNCHERS
// svsdf_cost_grad_multi (svsdf_kernels_multi.cuh).  launch_multi: what = 0 sparse / 1 batched k_outer_multi, 2 k_gsip_multi (grid <= 0:
// one full wave of the chosen variant); Z is read by the scaled units only.  The rigid units also run the pose table, the
// compaction and the finalize of every multi launch.
#define SVSDF_DECLARE_MULTI_LAUNCHERS(NS)                                                                         \
    namespace NS {                                                                                               \
    cudaError_t launch_multi(int what, const KernelArgs &A, const MultiArgs &M, const ShapeParams &S,            \
                             const ScaleSched *Z, int grid, size_t smem, int gsip_wide, int sm_count,            \
                             cudaStream_t st);                                                                   \
    }
SVSDF_DECLARE_MULTI_LAUNCHERS(fast_multi)
SVSDF_DECLARE_MULTI_LAUNCHERS(strict_multi)
SVSDF_DECLARE_MULTI_LAUNCHERS(fast_multi_scaled)
SVSDF_DECLARE_MULTI_LAUNCHERS(strict_multi_scaled)
#undef SVSDF_DECLARE_MULTI_LAUNCHERS
#define SVSDF_DECLARE_MULTI_RIGID(NS)                                                                            \
    namespace NS {                                                                                               \
    cudaError_t launch_pose_multi(double *blobs, const MultiArgs &M, int max_K1, cudaStream_t st);               \
    cudaError_t launch_compact_multi(const unsigned char *flag, int *list, const MultiArgs &M, cudaStream_t st); \
    cudaError_t launch_finalize_multi(const double *partials, const double *gsip_contrib, const int *gsip_piece, \
                                      const MultiArgs &M, int max_N, cudaStream_t st);                           \
    }
SVSDF_DECLARE_MULTI_RIGID(fast_multi)
SVSDF_DECLARE_MULTI_RIGID(strict_multi)
#undef SVSDF_DECLARE_MULTI_RIGID
cudaError_t launch_extract_count(const ExtractArgs &E, int *block_counts, int n_blocks, int64_t *n_total,
                                 cudaStream_t stream);
cudaError_t launch_extract_write(const ExtractArgs &E, const int *block_offsets, int n_blocks, double *out_xy,
                                 int64_t cap, cudaStream_t stream);
// svsdf_swept_contour (svsdf_swept.cu).  what: 0 classify + count per tile, 1 compact, 2 scatter the values (+ non-finite flag),
// 3 marching-squares counts, 4 emit vertices, 5 emit segments and triangles; scan: exclusive prefix of `channels` rows of n counts
// (row stride n + 1, the total lands at [n] and at totals[ch]) in one CTA.
cudaError_t launch_swept(int what, const SweptArgs &A, cudaStream_t st);
cudaError_t launch_swept_scan(int *counts, int n, int channels, int *totals, cudaStream_t st);
// svsdf_map_clearance (svsdf_clearance.cu).  what: 0 k_cl_count (band bits per word, band cells per CTA, occupied columns), 1 k_cl_write
// (the band's cells and centres in map order, after launch_swept_scan of the per-CTA counts).
cudaError_t launch_clearance(int what, const ClearanceArgs &A, cudaStream_t st);
// K5 (svsdf_frontend.cu)
cudaError_t launch_front_cells(const ShapeParams &S, const FrontParams &F, const double *yaws, unsigned char *cells, cudaStream_t st);
cudaError_t launch_front_expand(const ShapeParams &S, const FrontParams &F, const SubSwParams &P, const unsigned char *map,
                                const unsigned char *kbytes, int64_t n, const int *node_ij, const double *node_yaw, unsigned char *ok_out,
                                double *child_yaw_out, unsigned char *parts_out, cudaStream_t st);
// grid <= 0: no launch, *ctas_per_sm = resident k_astar_search CTAs per SM for this shape
cudaError_t launch_front_astar(const ShapeParams &S, const FrontParams &F, const SubSwParams &P, const unsigned char *map,
                               const unsigned char *kbytes, const AstarArgs &A, int grid, int *ctas_per_sm, cudaStream_t st);
cudaError_t launch_front_cspace(const FrontParams &F, const unsigned char *map, const unsigned *rowmask, unsigned *out, cudaStream_t st);
cudaError_t launch_front_check(const FrontParams &F, const unsigned char *map, const unsigned char *kbytes, int64_t n, const double *father_yaw,
                               const int *ind_xy, unsigned char *ok_out, double *child_yaw_out, cudaStream_t st);
}  // namespace svsdf
