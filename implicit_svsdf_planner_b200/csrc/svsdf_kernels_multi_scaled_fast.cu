// Multi-problem kernel translation unit for deformable robots (svsdf_set_scale), default (FMA contraction on) build: the scaled k_outer_multi /
// k_gsip_multi.  The pose-table, compaction and finalize kernels are shared with the rigid multi unit.
#define SVSDF_NS fast_multi_scaled
#define SVSDF_SCALED_UNIT 1
#define SVSDF_MULTI_UNIT 1
#include "svsdf_kernels_multi.cuh"
