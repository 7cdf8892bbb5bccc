// Multi-problem kernel translation unit (svsdf_cost_grad_multi), default (FMA contraction on) build: k_outer_multi / k_gsip_multi and the pose-table,
// compaction and finalize kernels of a multi-problem evaluation.  Kept apart from the single-problem units so that those compile as
// they did.
#define SVSDF_NS fast_multi
#define SVSDF_MULTI_UNIT 1
#include "svsdf_kernels_multi.cuh"
