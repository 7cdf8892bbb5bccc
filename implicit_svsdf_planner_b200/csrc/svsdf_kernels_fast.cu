// Kernel translation unit, default build: FMA contraction enabled (nvcc default -fmad=true).  The single-problem cost kernels of a rigid
// robot and the kernels every single-problem variant shares.
#define SVSDF_NS fast
#define SVSDF_SCALED 0
#include "svsdf_kernels_single.cuh"
#include "svsdf_kernels_shared.cuh"
