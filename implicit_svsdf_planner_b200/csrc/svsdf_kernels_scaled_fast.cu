// Kernel translation unit for deformable robots (svsdf_set_scale), default build: FMA contraction enabled.  Only the
// scaled k_outer / k_gsip instantiations live here, so they compile in parallel with the rigid units and leave them as
// they are.
#define SVSDF_NS fast_scaled
#define SVSDF_SCALED 1
#include "svsdf_kernels_single.cuh"
