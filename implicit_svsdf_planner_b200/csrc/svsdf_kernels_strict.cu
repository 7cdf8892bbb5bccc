// Kernel translation unit, parity-debug build: compiled with -fmad=false so every a*b+c rounds twice like the
// CPU oracle / the reference's x86-64 build (SURVEY.md §7 "Hard parts").  The single-problem cost kernels of a rigid robot and the
// kernels every single-problem variant shares.
#define SVSDF_NS strict
#define SVSDF_SCALED 0
#include "svsdf_kernels_single.cuh"
#include "svsdf_kernels_shared.cuh"

#ifdef SVSDF_PHASE_STATS
// scripts/outer_phase_stats.py: where the batched k_outer of this unit writes its per-warp counters ([8 x grid][6] 64-bit words)
extern "C" int svsdf_phase_stats_buffer(unsigned long long *buf) {
    return (int)cudaMemcpyToSymbol(svsdf::strict::g_phase_stats, &buf, sizeof(buf));
}
#endif
