// Kernel translation unit for deformable robots (svsdf_set_scale), parity build: compiled with -fmad=false like
// svsdf_kernels_strict.cu, so the scaled path rounds like the CPU oracle.  Only the scaled k_outer / k_gsip instantiations.
#define SVSDF_NS strict_scaled
#define SVSDF_SCALED 1
#include "svsdf_kernels_single.cuh"
