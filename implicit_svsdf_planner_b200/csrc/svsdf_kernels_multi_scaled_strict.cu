// Multi-problem kernel translation unit for deformable robots (svsdf_set_scale), parity (-fmad=false) build: the scaled k_outer_multi /
// k_gsip_multi.  The pose-table, compaction and finalize kernels are shared with the rigid multi unit.
#define SVSDF_NS strict_multi_scaled
#define SVSDF_SCALED 1
#include "svsdf_kernels_multi.cuh"
