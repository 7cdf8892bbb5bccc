// Multi-problem kernel translation unit (svsdf_cost_grad_multi), parity (-fmad=false) build: k_outer_multi / k_gsip_multi and the pose-table,
// compaction and finalize kernels of a multi-problem evaluation.  Kept apart from the single-problem units so that those compile as
// they did.
#define SVSDF_NS strict_multi
#define SVSDF_SCALED 0
#include "svsdf_kernels_multi.cuh"
#include "svsdf_kernels_multi_shared.cuh"
