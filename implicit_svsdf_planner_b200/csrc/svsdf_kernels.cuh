// svsdf_kernels.cuh — sm_90a (H100) kernels for the SVSDF collision cost + gradient hot path.
//
// Replaces the OpenMP loop  TrajOptimizer::addSaftyPenaOnSweptVolumeParallelTrueSDF
// (src/planner_algorithm/include/planner_algorithm/back_end_optimizer.hpp:774-869) and everything it calls in
// SweptVolumeManager (src/swept_volume/include/swept_volume/sw_manager.hpp:465-474, 521-526, 538-581, 741-757,
// 779-806, 844-866, 916-1018, 1249-1325).
//
// Mapping (one warp per query point):
//   * the trajectory blob (durations, quintic coefficients, layer-1 time lattice and its pose table) is pulled
//     into shared memory once per CTA with a TMA bulk copy (cp.async.bulk + mbarrier);
//   * choiceTInit's four scan layers are evaluated 32 samples per round, one sample per lane, and reduced with
//     a shuffle arg-min that keeps the reference's "first strict minimum wins" rule;
//   * gradientDescent's inner loop (29 step halvings, each needing 3 SDF evaluations) is evaluated
//     speculatively in parallel: lanes 30/31 compute the finite-difference slope, lanes 0-29 the candidates for
//     both signs, and the first accepted halving is picked with a ballot — decisions are identical to the
//     sequential loop given identical SDF values;
//   * the FD gradient uses 4 lanes; the smoothed-L1 penalty and the chain rule to the 6x3 coefficient block are
//     accumulated in per-warp shared-memory accumulators (no atomics), reduced per CTA in a fixed order and
//     written as one partial per CTA; a tiny finalize kernel sums the partials in a fixed order, so results are
//     bit-reproducible run to run.
//   * points found inside the swept volume (sdf <= 0) are compacted in index order and handled by k_gsip, one
//     CTA per point, ring samples spread over the CTA's warps.
//
// This file holds what every cost unit compiles: the device code and the kernel templates of k_outer / k_gsip, and the launch
// helpers their launchers share.  Each unit (svsdf_kernels{,_scaled,_multi,_multi_scaled}_{fast,strict}.cu) includes it through the
// launchers it carries: svsdf_kernels_single.cuh or svsdf_kernels_multi.cuh, and in the rigid units the kernels the scaled ones share
// (svsdf_kernels_shared.cuh, svsdf_kernels_multi_shared.cuh).  Every unit is compiled with FMA contraction (fast) and with
// -fmad=false ("strict": same rounding sequence as the CPU, used to debug parity).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "svsdf_shapes.cuh"
#include "svsdf_sincos.cuh"
#include "svsdf_types.h"

#ifndef SVSDF_NS
#error "define SVSDF_NS (fast|strict) before including svsdf_kernels.cuh"
#endif

namespace svsdf {
namespace SVSDF_NS {

constexpr unsigned FULL = 0xffffffffu;
using dev::smaxd;
using dev::smind;

// SVSDF_PHASE_STATS (scripts/outer_phase_stats.py builds the strict unit with it; never defined in the product): the batched
// k_outer counts, per warp, the descent's issued and useful lane-evaluations and the clock64() cycles of its phases into
// g_phase_stats[8 blockIdx.x + warp][6]: issued, useful, then cycles of the seed scan (up to the barrier that opens the queue), the
// descent, the wait at the barrier after it, and the gradient + epilogue + accumulation.  Without the macro none of it exists.
#ifdef SVSDF_PHASE_STATS
#define SVSDF_STATS(...) __VA_ARGS__
#define SVSDF_STATS_PARAM(...) , __VA_ARGS__
__device__ unsigned long long *g_phase_stats = nullptr;
#else
#define SVSDF_STATS(...)
#define SVSDF_STATS_PARAM(...)
#endif

// ------------------------------------------------------------------------------------------------
// Trajectory view over the shared-memory copy of the blob
// ------------------------------------------------------------------------------------------------
struct TrajView {
    int N, K1;
    double D;
    const double *T;     // [N]
    const double *c;     // [N][3][6] ascending powers
    const double *lat;   // [K1]
    const double *pose;  // [4][K1pad] SoA: x, y, cos, sin
    int K1pad;
    // the same arrays as 32-bit shared-window addresses (valid when the view is on the shared-memory copy of the blob):
    // the hot loops read through these with ld.shared so the address is one register + immediate instead of a
    // generic pointer whose shared-window base the compiler re-derives (S2R SR_CgaCtaId + LEA) at every use
    uint32_t sT, sc, slat, spose;
};

__device__ __forceinline__ double lds_f64(uint32_t a) {
    double v;
    asm("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ void lds_v2(uint32_t a, double &v0, double &v1) {
    asm("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(v0), "=d"(v1) : "r"(a));
}

__device__ __forceinline__ TrajView make_view(const double *blob) {
    TrajView tv;
    tv.N = (int)blob[0];
    tv.K1 = (int)blob[1];
    tv.D = blob[2];
    BlobLayout L = blob_layout(tv.N, tv.K1);
    tv.T = blob + L.off_T;
    tv.c = blob + L.off_c;
    tv.lat = blob + L.off_lat;
    tv.pose = blob + L.off_pose;
    tv.K1pad = L.K1pad;
    // (meaningless for a view on global memory, k_pose_table).  The blob is read-only once the TMA copy has landed; the
    // empty volatile asm orders every ld.shared that derives its address from `sb` after the mbarrier wait.
    uint32_t sb = (uint32_t)__cvta_generic_to_shared(blob);
    asm volatile("" : "+r"(sb) : : "memory");
    tv.sT = sb + 8u * (uint32_t)L.off_T;
    tv.sc = sb + 8u * (uint32_t)L.off_c;
    tv.slat = sb + 8u * (uint32_t)L.off_lat;
    tv.spose = sb + 8u * (uint32_t)L.off_pose;
    return tv;
}

// Trajectory<5>::locatePieceIdx (trajectory.hpp:498-516): subtract durations while t > dur (strict).
__device__ __forceinline__ int locate_piece(const TrajView &tv, double &t) {
    int idx = 0;
#pragma unroll 1
    for (; idx < tv.N; ++idx) {
        double dur = tv.T[idx];
        if (!(t > dur)) break;
        t -= dur;
    }
    if (idx == tv.N) {
        idx--;
        t += tv.T[idx];
    }
    return idx;
}

// locatePieceIdx with a guess.  The reference's loop yields piece h and local time t_h = ((t - T_0) - T_1) ... - T_{h-1}
// (one rounding per subtraction) iff every test before h passed and the test at h failed.  fl(a - b) > 0 <=> a > b, so
// "all earlier tests passed" is equivalent to t_h > 0 (induction: t_h > 0 => t_{h-1} > T_{h-1} > 0 => ...).  With the
// guess taken from the caller's previous sample (consecutive samples of a scan or of a descent almost always fall into
// the same piece) the search is the bare subtraction chain plus two compares; a wrong guess (or NaN, or the idx == N
// wrap-around case) falls back to the reference loop.  Same result bit for bit.
__device__ __forceinline__ int locate_piece(const TrajView &tv, double &t, int &hint) {
    const int h = hint;
    double tl = t;
    uint32_t a = tv.sT;  // 16-byte aligned
    int i = 0;
#pragma unroll 1
    for (; i + 2 <= h; i += 2, a += 16) {
        double d0, d1;
        lds_v2(a, d0, d1);
        tl -= d0;
        tl -= d1;
    }
    if (i < h) {
        tl -= lds_f64(a);
        a += 8;
    }
    const double Th = lds_f64(a);  // T[h]
    if ((h == 0 || tl > 0.0) && !(tl > Th)) {
        t = tl;
        return h;
    }
    hint = locate_piece(tv, t);
    return hint;
}

// Piece<5>::getPos (trajectory.hpp:104-114): ascending powers with tn *= t (not Horner).
__device__ __forceinline__ void traj_pos_at(const TrajView &tv, int i, double t, double &x, double &y, double &yaw) {
    const uint32_t a = tv.sc + 144u * (uint32_t)i;  // 18 doubles per piece, 16-byte aligned
    double c[18];
#pragma unroll
    for (int k = 0; k < 9; ++k) lds_v2(a + 16u * k, c[2 * k], c[2 * k + 1]);
    x = 0.0; y = 0.0; yaw = 0.0;
    double tn = 1.0;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        x += tn * c[k];
        y += tn * c[6 + k];
        yaw += tn * c[12 + k];
        tn *= t;
    }
}
__device__ __forceinline__ void traj_pos(const TrajView &tv, double t, double &x, double &y, double &yaw) {
    int i = locate_piece(tv, t);
    const double *c = tv.c + 18 * i;
    x = 0.0; y = 0.0; yaw = 0.0;
    double tn = 1.0;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        x += tn * c[k];
        y += tn * c[6 + k];
        yaw += tn * c[12 + k];
        tn *= t;
    }
}

// Piece<5>::getVel (trajectory.hpp:116-128)
__device__ __forceinline__ void traj_vel(const TrajView &tv, double t, double &vx, double &vy, double &vw) {
    int i = locate_piece(tv, t);
    const double *c = tv.c + 18 * i;
    vx = 0.0; vy = 0.0; vw = 0.0;
    double tn = 1.0;
#pragma unroll
    for (int k = 1; k < 6; ++k) {
        double f = (double)k * tn;
        vx += f * c[k];
        vy += f * c[6 + k];
        vw += f * c[12 + k];
        tn *= t;
    }
}

// getStateOnTrajStamp (sw_manager.hpp:465-474) + posEva2Rel (:521-526): rel = Rz(yaw)^T (p - x)
__device__ __forceinline__ void rel_from_pose(double px, double py, double x, double y, double cy, double sy,
                                              double &rx, double &ry) {
    double d0 = px - x, d1 = py - y;
    rx = cy * d0 + sy * d1;
    ry = -sy * d0 + cy * d1;
}

// one record of the pose windows (read-only during the kernel that reads it): two 16-byte loads of one 32-byte sector
__device__ __forceinline__ PoseRec ld_pose(const PoseRec *p) {
    const double2 a = __ldg(reinterpret_cast<const double2 *>(p)), b = __ldg(reinterpret_cast<const double2 *>(p) + 1);
    PoseRec r;
    r.x = a.x; r.y = a.y; r.c = b.x; r.s = b.y;
    return r;
}

// Deformable robot (useScale == true): getScale(t) = diag(sx, sy, 1) (ScaleSched) and the diagonal (ix, iy) of St.inverse()
// by Eigen 3.3's size-3 cofactor formula: 1/det with det = sy * sx, then ix = sy * (1/det), iy = sx * (1/det) — not 1/sx.
// t is the absolute time of the sample.
__device__ __forceinline__ void scale_inv(const ScaleSched &Z, double t, double &ix, double &iy) {
    double s0, c0, s1, c1;
    dev::sincos_portable(Z.w[0] * t + Z.phi[0], s0, c0);
    dev::sincos_portable(Z.w[1] * t + Z.phi[1], s1, c1);
    const double sx = Z.a[0] + s0 * Z.b[0], sy = Z.a[1] + s1 * Z.b[1];
    const double inv = 1.0 / (sy * sx);
    ix = sy * inv;
    iy = sx * inv;
}
// posEva2Rel(p, xt, Rt, St) (sw_manager.hpp:528-535): rel = (Rt^T St^-1) (p - xt), the 3x3 product first (eager Eigen):
// its 2x2 block is [[c ix, s iy], [-s ix, c iy]].  SCALED == false: rel_from_pose, Z unused.
template <bool SCALED>
__device__ __forceinline__ void rel_at(const ScaleSched *Z, double t, double px, double py, double x, double y, double cy,
                                       double sy, double &rx, double &ry) {
    if constexpr (SCALED) {
        double ix, iy;
        scale_inv(*Z, t, ix, iy);
        const double d0 = px - x, d1 = py - y;
        rx = (cy * ix) * d0 + (sy * iy) * d1;
        ry = (-sy * ix) * d0 + (cy * iy) * d1;
    } else {
        rel_from_pose(px, py, x, y, cy, sy, rx, ry);
    }
}

// getSDFAtTimeStamp<SCALED> (sw_manager.hpp:741-757; the mesh functor's _igl variant :760-777)
template <int SHAPE, bool XFORM, bool SCALED = false>
__device__ __forceinline__ double eval_sdf(const TrajView &tv, const ShapeParams &S, double px, double py, double t,
                                           const ScaleSched *Z = nullptr) {
    double x, y, yaw, sy, cy, rx, ry;
    const double ta = t;
    traj_pos(tv, t, x, y, yaw);
    dev::sincos_portable(yaw, sy, cy);
    rel_at<SCALED>(Z, ta, px, py, x, y, cy, sy, rx, ry);
    return dev::shape_sdf<SHAPE, XFORM>(S, rx, ry);
}
// same with a piece-index guess carried by the caller from its previous sample
template <int SHAPE, bool XFORM, bool SCALED = false>
__device__ __forceinline__ double eval_sdf(const TrajView &tv, const ShapeParams &S, double px, double py, double t, int &hint,
                                           const ScaleSched *Z = nullptr) {
    double x, y, yaw, sy, cy, rx, ry;
    const double ta = t;  // absolute time: locate_piece makes t piece-local
    const int i = locate_piece(tv, t, hint);
    traj_pos_at(tv, i, t, x, y, yaw);
    dev::sincos_portable(yaw, sy, cy);
    rel_at<SCALED>(Z, ta, px, py, x, y, cy, sy, rx, ry);
    return dev::shape_sdf<SHAPE, XFORM>(S, rx, ry);
}

// Warp arg-min with the sequential loop's semantics: the FIRST lane holding the minimum value wins; NaN never wins
// (callers map NaN to +inf; the reference's test is `dis < min_dis`).  Two 32-bit REDUX.MIN over an order-preserving
// integer image of the double, then a ballot for the first lane.  Returns the winning lane; f becomes the minimum.
__device__ __forceinline__ int warp_argmin_lane(double &f) {
    f = f + 0.0;  // -0.0 -> +0.0 so that equal values have equal keys
    unsigned long long b = (unsigned long long)__double_as_longlong(f);
    b ^= (b >> 63) ? 0xffffffffffffffffull : 0x8000000000000000ull;  // monotone map double -> uint64
    const unsigned hi = (unsigned)(b >> 32), lo = (unsigned)b;
    const unsigned mh = __reduce_min_sync(FULL, hi);
    const unsigned ml = __reduce_min_sync(FULL, hi == mh ? lo : 0xffffffffu);
    const unsigned win = __ballot_sync(FULL, hi == mh && lo == ml);
    const int src = __ffs(win) - 1;
    f = __shfl_sync(FULL, f, src);
    return src;
}

struct OuterResult {
    double sdf, tstar;
    int evals;  // lane-evaluations executed (active lanes), for E_executed accounting
};

// getSDFofSweptVolume<false,*> (sw_manager.hpp:844-866) = choiceTInit (:538-581) + gradientDescent (:1249-1325),
// executed cooperatively by one warp. All lanes return the same values.
//
// After the table-driven layer 1 and the three 21-sample layers of choiceTInit, the descent is organised as ROUNDS of one
// SDF evaluation per lane, driven by a small warp-uniform state machine with a single eval_sdf call site:
//   M_F0   f(x0) when no sample was below the initial 1e9 (degenerate input; the reference evaluates it at iter == 0)
//   M_A    first descent step: lanes 0-14 x - tau_j (slope sign +1), 15-29 x + tau_j (sign -1), j = 0..14; 30/31 slope
//   M_B    halvings j = 15..28 in the known direction (only if M_A found no decreasing candidate)
//   M_P    29 halvings in the PREDICTED direction + slope on lanes 30/31
//   M_M    29 halvings in the actual direction after a misprediction
// Decisions are the sequential loop's: the slope's sign always comes from the finite difference on lanes 30/31, and the
// accepted halving is the first (largest step) whose candidate decreases f.
// SCALED (deformable robot, schedule *Z): only the descent evaluates the scaled shape; choiceTInit's 2-argument overload
// (:538-581) never reads its template flag, so the four seed layers stay rigid.
// w2 / w3: the pose windows of layers 2 and 3 (thread_choice_t_init); null: the layer evaluates the trajectory.
template <int SHAPE, bool XFORM, bool SCALED = false>
__device__ __forceinline__ OuterResult solve_outer(const TrajView &tv, const ShapeParams &S, double px, double py,
                                                   const PoseRec *w2, const PoseRec *w3, bool have_seed = false,
                                                   double seed_in = 0.0, double min_in = 1e9, const ScaleSched *Z = nullptr) {
    const int lane = threadIdx.x & 31;
    const double D = tv.D;
    const double INF = __longlong_as_double(0x7ff0000000000000LL);
    int evals = 0;

    // ---- choiceTInit layer 1: shared lattice t_k (accumulated 0.15 adds) with the pose table ----
    // Exact pruning as in thread_choice_t_init: the result is the lexicographic minimum of (f_k, k) over the samples with
    // f_k < 1e9, and f_k >= |p - x_k| - S.rout.  The 32 lattice poses around the one nearest to p are evaluated first (one
    // round: this already contains the minimum almost always), then every block of 32 is revisited and only samples with
    // |p - x_k| <= min + rout are evaluated (usually none).  (Skipped when the caller ran choiceTInit thread-per-point.)
    double min_dis = have_seed ? min_in : 1e9, seed = have_seed ? seed_in : 0.0;
    int kb = -1;
    if (!have_seed) {
        const uint32_t row = 8u * (uint32_t)tv.K1pad;
        const int K1 = tv.K1;
        // nearest lattice pose
        double bd2 = INF;
        int k0 = 0;
        for (int k = lane; k < K1; k += 32) {
            const uint32_t ps = tv.spose + 8u * (uint32_t)k;
            const double ax = px - lds_f64(ps), ay = py - lds_f64(ps + row);
            const double d2 = ax * ax + ay * ay;
            if (d2 < bd2) { bd2 = d2; k0 = k; }
        }
        {
            double v = bd2;
            const int src = warp_argmin_lane(v);
            k0 = __shfl_sync(FULL, k0, src);
        }
        const int w0 = max(0, min(k0 - 16, K1 - 32));   // window [w0, w0 + 32) (whole lattice when K1 <= 32)
        double thr2 = INF;
        // it = -1: the window; it >= 0: block it (samples of the window are not evaluated twice)
        for (int it = -1; 32 * it < K1; ++it) {
            const int k = (it < 0) ? w0 + lane : 32 * it + lane;
            bool need = k >= 0 && k < K1;
            double rx = 0.0, ry = 0.0;
            if (need) {
                const uint32_t ps = tv.spose + 8u * (uint32_t)k;
                const double xk = lds_f64(ps), yk = lds_f64(ps + row);
                const double ax = px - xk, ay = py - yk;
                need = (it < 0) || ((ax * ax + ay * ay <= thr2) && !(k >= w0 && k < w0 + 32));
                if (need) rel_from_pose(px, py, xk, yk, lds_f64(ps + 2 * row), lds_f64(ps + 3 * row), rx, ry);
            }
            const unsigned mneed = __ballot_sync(FULL, need);
            if (mneed == 0u) continue;
            double f = INF;
            if (need) {
                f = dev::shape_sdf<SHAPE, XFORM>(S, rx, ry);
                if (!(f == f)) f = INF;
            }
            evals += __popc(mneed);
            const int kl = k - lane + warp_argmin_lane(f);   // first lane holding the block minimum; f := that minimum
            if (__any_sync(FULL, f < min_dis || (f == min_dis && f < 1e9 && kl < kb))) {
                min_dis = f;
                kb = kl;
                const double thr0 = f * S.prune_scale + S.rout, thr = fmax(thr0, S.prune_rmin);  // analytic shapes: f * 1 + rout, max with 0
                thr2 = (thr0 >= 0.0) ? thr * thr : INF;
            }
        }
        seed = (kb >= 0) ? lds_f64(tv.slat + 8u * (uint32_t)kb) : 0.0;
    }

    // ---- choiceTInit layers 2..4: 21-sample window around the seed, dt *= 0.1 per layer, one sample per lane ----
    if (!have_seed) {
        double dt = 0.15;
        int hint = 0;
        // layers 2 and 3: lane m reads sample m's pose from the window of kb (layer 2) or of (kb, m2) (layer 3) when it is built
        const PoseRec *win = w2 ? w2 + kWinLen * (kb + 1) : nullptr;
        int m2 = -1;
#pragma unroll 1
        for (int layer = 2; layer <= 4; ++layer) {
            dt *= 0.1;
            double t = smaxd(0.0, seed - 10 * dt);
            const double term = smind(D, seed + 10 * dt);
#pragma unroll
            for (int i = 0; i < 20; ++i)
                if (i < lane) t += dt;  // lane k (<= 20) holds t0 + dt added k times (same rounding as the loop)
            double fq;
            if (win) {
                const PoseRec ps = ld_pose(win + min(lane, kWinLen - 1));
                double rx, ry;
                rel_from_pose(px, py, ps.x, ps.y, ps.c, ps.s, rx, ry);
                fq = dev::shape_sdf<SHAPE, XFORM>(S, rx, ry);
            } else {
                fq = eval_sdf<SHAPE, XFORM>(tv, S, px, py, t, hint);
            }
            const bool lat_valid = (lane <= 20) && (t <= term);
            double fl = (lat_valid && (fq == fq)) ? fq : INF;
            evals += __popc(__ballot_sync(FULL, lat_valid));
            const int src = warp_argmin_lane(fl);  // fl := warp minimum
            const double tb = __shfl_sync(FULL, t, src);
            if (__any_sync(FULL, fl < min_dis)) {
                min_dis = fl;
                seed = tb;
                if (layer == 2) m2 = src;
            }
            win = (layer == 2 && w3) ? w3 + kWinLen * (kWin3Stride * (kb + 1) + m2 + 1) : nullptr;
        }
    }

    // ---- gradientDescent (:1249-1325) from x0 = seed, bounds [ts-3.4, ts+3.4] ∩ [0, D] (:856-857) ----
    // ROUNDS of one evaluation per lane.  Per-lane round constants: tau (step of this lane's candidate), sbit (sign bit
    // of the offset: candidates move against the slope direction the round assumes) and the clamp interval — the
    // descent interval for candidates, [0, +inf) / (-inf, D] for the two finite-difference samples on lanes 30 / 31
    // (smaxd(0, x - 1e-6), smind(D, x + 1e-6): :798-806).  They change only when the round type changes.
    enum { M_F0 = 0, M_A, M_B, M_P, M_M };
    const double t_min = smaxd(0.0, seed - 3.4), t_max = smind(seed + 3.4, D);
    const bool slope_lane = lane >= 30;
    const double lo_l = slope_lane ? (lane == 30 ? 0.0 : -INF) : t_min;
    const double hi_l = slope_lane ? (lane == 30 ? INF : D) : t_max;
    const int hi001 = __double2hiint(0.01), lo001 = __double2loint(0.01);
    // alpha = 0.01 halved j times: exact, so subtract j from the exponent field (0.01 * 2^-46 is still normal)
    const int tauP_hi = slope_lane ? __double2hiint(0.000001) : hi001 - (lane << 20);
    const int tau_lo = slope_lane ? __double2loint(0.000001) : lo001;
    const unsigned sbit_fix = (lane == 30) ? 0x80000000u : 0u;  // lane 30: x - 1e-6, lane 31: x + 1e-6
    double x = seed, fx = min_dis, prev_x = 10000000.0;
    int iter = 0, pred = 0, sgn = 0, hint = 0;
    int mode;
    int tau_hi;        // this lane's step, high word
    unsigned sbit;     // this lane's offset sign bit
    // SCALED: the reference evaluates f(x0) at iter == 0 with the scaled shape, which is not the rigid seed minimum
    if (SCALED || __any_sync(FULL, min_dis >= 1e9)) {
        // nothing below the initial 1e9 (degenerate input): the reference evaluates f(x0) at iter == 0
        mode = M_F0;
        tau_hi = 0; sbit = 0;   // offset +0.0: the sample is x itself
    } else {
        mode = M_A;
        prev_x = x;             // `prev_x = x` after the (true) first loop test
        tau_hi = slope_lane ? tauP_hi : hi001 - (((lane < 15) ? lane : lane - 15) << 20);
        sbit = slope_lane ? sbit_fix : ((lane < 15) ? 0x80000000u : 0u);
    }
    bool running = true;
#pragma unroll 1
    while (running) {
        const double off = __hiloint2double(tau_hi ^ (int)sbit, (mode == M_F0) ? 0 : tau_lo);
        const double tq = smaxd(smind(x + off, hi_l), lo_l);
        const double fq = eval_sdf<SHAPE, XFORM, SCALED>(tv, S, px, py, tq, hint, Z);
        const unsigned m_dec = __ballot_sync(FULL, (fq - fx) < 0);  // candidates that decrease f
        int jacc = -1, src = 0;
        bool failed = false, step_end = true;
        if (mode == M_P) {
            // 29 halvings in the predicted direction + the slope: the common round
            evals += 31;
            const double g = (__shfl_sync(FULL, fq, 31) - __shfl_sync(FULL, fq, 30)) * 500000;
            sgn = (int)__any_sync(FULL, g > 0) - (int)__any_sync(FULL, g < 0);  // (int)(g > 0) - (g < 0)
            const unsigned m = m_dec & 0x1fffffffu;
            if (sgn != 0 && sgn != pred) {  // mispredicted: redo the halvings in the actual direction
                mode = M_M;
                sbit = (sgn > 0) ? 0x80000000u : 0u;
                step_end = false;
            } else if (sgn != 0 && m) {
                jacc = __ffs(m) - 1; src = jacc;
            } else failed = true;
        } else if (mode == M_M) {
            evals += 29;
            const unsigned m = m_dec & 0x1fffffffu;
            if (m) { jacc = __ffs(m) - 1; src = jacc; }
            else failed = true;
        } else if (mode == M_A) {
            // first step: lanes 0-14 x - tau_j (slope sign +1), 15-29 x + tau_j (sign -1), j = 0..14; 30/31 slope
            evals += 32;
            const double g = (__shfl_sync(FULL, fq, 31) - __shfl_sync(FULL, fq, 30)) * 500000;
            sgn = (int)__any_sync(FULL, g > 0) - (int)__any_sync(FULL, g < 0);
            const unsigned grp = (sgn > 0) ? (m_dec & 0x7fffu) : ((m_dec >> 15) & 0x7fffu);
            if (sgn == 0) failed = true;
            else if (grp) { jacc = __ffs(grp) - 1; src = (sgn > 0) ? jacc : jacc + 15; }
            else {  // halvings j = 15..28 in the known direction
                mode = M_B;
                tau_hi = hi001 - ((15 + lane) << 20);
                sbit = (sgn > 0) ? 0x80000000u : 0u;
                step_end = false;
            }
        } else if (mode == M_B) {
            evals += 14;
            const unsigned mb = m_dec & 0x3fffu;
            if (mb) { src = __ffs(mb) - 1; jacc = 15 + src; }
            else failed = true;
        } else {  // M_F0
            fx = __shfl_sync(FULL, fq, 0);
            evals += 1;
        }
        if (jacc >= 0) {
            const double xacc = __shfl_sync(FULL, tq, src), facc = __shfl_sync(FULL, fq, src);
            // a full, unclamped stride means we are still walking downhill: same slope sign next; otherwise the step
            // overshot the minimiser (tau_j is the largest decreasing step) and the slope flips
            const bool walking = (jacc == 0) && __all_sync(FULL, xacc == x + (-0.01 * (double)sgn));
            pred = walking ? sgn : -sgn;
            x = xacc;
            fx = facc;
            iter += jacc + 1;
        } else if (failed) {
            iter += 29;
        }
        if (step_end) {
            // while (iter < max_iter && !stop && abs(x - prev_x) > tol)   (:1288)
            running = (iter < 1000) && !failed && __all_sync(FULL, fabs(x - prev_x) > 1e-16);
            prev_x = x;
            if (pred == 0) {  // only after M_F0: first descent step
                mode = M_A;
                tau_hi = slope_lane ? tauP_hi : hi001 - (((lane < 15) ? lane : lane - 15) << 20);
                sbit = slope_lane ? sbit_fix : ((lane < 15) ? 0x80000000u : 0u);
            } else {
                mode = M_P;
                tau_hi = tauP_hi;
                sbit = slope_lane ? sbit_fix : ((pred > 0) ? 0x80000000u : 0u);
            }
        }
    }
    OuterResult R;
    R.sdf = fx;
    R.tstar = x;
    R.evals = evals;
    return R;
}

// getGradPrelAtTimeStamp (sw_manager.hpp:779-795) -> getonlyGrad1: central FD, dx = 1e-6 in the body frame
// (Shape.hpp:35-53), or the Polygon's analytic override (Shape.hpp:1508-1534). 4 lanes do the 4 evaluations.
template <int SHAPE, bool XFORM, bool SCALED = false>
__device__ __forceinline__ void grad_prel(const TrajView &tv, const ShapeParams &S, double px, double py, double t,
                                          double &gx, double &gy, const ScaleSched *Z = nullptr) {
    const int lane = threadIdx.x & 31;
    double x, y, yaw, sy, cy, rx, ry;
    traj_pos(tv, t, x, y, yaw);
    dev::sincos_portable(yaw, sy, cy);
    rel_at<SCALED>(Z, t, px, py, x, y, cy, sy, rx, ry);
    if (SHAPE == SH_POLYGON) {
        dev::PolyHit H = dev::polygon_scan(S, rx, ry);
        double vx = rx - H.cx, vy = ry - H.cy;
        double z = vx * vx + vy * vy;
        if (z > 0.0) {
            double n = sqrt(z);
            vx /= n; vy /= n;
        }
        if (H.rs % 2 != 0) { vx = -vx; vy = -vy; }
        gx = vx; gy = vy;
        return;
    }
    if (SHAPE == SH_CIRCLE) {
        dev::circle_grad1<XFORM>(S, rx, ry, gx, gy);
        return;
    }
    const double dx = 0.000001;
    double qx = rx, qy = ry;
    if (lane == 0) { qx -= dx; }
    if (lane == 1) { qx -= dx; qx += 2 * dx; }
    if (lane == 2) { qy -= dx; }
    if (lane == 3) { qy -= dx; qy += 2 * dx; }
    double f = dev::shape_sdf<SHAPE, XFORM>(S, qx, qy);
    double f0 = __shfl_sync(FULL, f, 0), f1 = __shfl_sync(FULL, f, 1);
    double f2 = __shfl_sync(FULL, f, 2), f3 = __shfl_sync(FULL, f, 3);
    gx = (f1 - f0) / (2 * dx);
    gy = (f3 - f2) / (2 * dx);
}

// smoothedL1 (back_end_optimizer.hpp:316-340), mu = 0.01
__device__ __forceinline__ bool smoothed_l1(double x, double mu, double &f, double &df) {
    if (x < 0.0) return false;
    if (x > mu) {
        f = x - 0.5 * mu;
        df = 1.0;
        return true;
    }
    const double xdmu = x / mu;
    const double sqrxdmu = xdmu * xdmu;
    const double mumxd2 = mu - 0.5 * x;
    f = mumxd2 * sqrxdmu * xdmu;
    df = sqrxdmu * ((-0.5) * xdmu + 3.0 * mumxd2 / mu);
    return true;
}

// Per-point penalty and chain rule: the loop body of addSaftyPenaOnSweptVolumeParallelTrueSDF after the SDF
// query (back_end_optimizer.hpp:797-854) with grad_cost_p_sw (:1031-1066).
// In: world point p, sdf, t*, gradient g (body frame for sdf > 0; world-frame GSIP direction otherwise).
// Out (uniform across the warp): piece index, beta0[6], G[3] = w_p * (d/dx, d/dy, d/dyaw), gdT, pena.
struct Contribution {
    int piece;
    double s1;
    double G[3];
    double gdT, pena;
    bool active;
};
// SCALED: sdf_grad = -L' (-(St^-1)^T rotate g) with St = getScale(t*) at the absolute t* (:827, :1050); the yaw term keeps
// the reference's form without St^-1 (:1062; exact only at St = I) and gdT has no dS/dt term (at fixed t*, S does not
// depend on the durations).
template <bool SCALED = false>
__device__ __forceinline__ Contribution point_contribution(const TrajView &tv, const CostParams &cp, double px,
                                                           double py, double sdf, double tstar, double gx,
                                                           double gy, const ScaleSched *Z = nullptr) {
    Contribution C;
    double tl = tstar;
    int i = locate_piece(tv, tl);
    const double *c = tv.c + 18 * i;
    double s1 = tl, s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2, s5 = s4 * s1;
    double b0[6] = {1.0, s1, s2, s3, s4, s5};
    double b1[6] = {0.0, 1.0, 2.0 * s1, 3.0 * s2, 4.0 * s3, 5.0 * s4};
    double pos[3], vel[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int q = 0; q < 6; ++q) {
            a += c[6 * d + q] * b0[q];
            b += c[6 * d + q] * b1[q];
        }
        pos[d] = a;
        vel[d] = b;
    }
    double yaw = pos[2], sy, cy;
    dev::sincos_portable(yaw, sy, cy);
    if (sdf < 0) {  // :832 world -> body
        double g0 = cy * gx + sy * gy;
        double g1 = -sy * gx + cy * gy;
        gx = g0; gy = g1;
    }
    double sdf_cost = -1.0, sdf_out_grad = 0.0;
    smoothed_l1(cp.safety_hor - sdf, 0.01, sdf_cost, sdf_out_grad);
    C.piece = i;
    C.s1 = s1;
    C.G[0] = C.G[1] = C.G[2] = 0.0;
    C.gdT = 0.0;
    C.pena = 0.0;
    C.active = false;
    if (sdf_cost > 0) {
        double rg0, rg1;
        if constexpr (SCALED) {
            double ix, iy;
            scale_inv(*Z, tstar, ix, iy);
            rg0 = -((ix * cy) * gx + (-(ix * sy)) * gy);
            rg1 = -((iy * sy) * gx + (iy * cy) * gy);
        } else {
            rg0 = -(cy * gx + (-sy) * gy);
            rg1 = -(sy * gx + cy * gy);
        }
        double sg0 = -sdf_out_grad * rg0, sg1 = -sdf_out_grad * rg1;
        double d0 = px - pos[0], d1 = py - pos[1];
        double w0 = -sy * d0 + cy * d1;
        double w1 = -cy * d0 + -sy * d1;
        double gyaw = (-sdf_out_grad * gx) * w0 + (-sdf_out_grad * gy) * w1;
        C.G[0] = cp.weight_p * sg0;
        C.G[1] = cp.weight_p * sg1;
        C.G[2] = cp.weight_p * gyaw;
        C.pena = cp.weight_p * sdf_cost;
        C.gdT = -(C.G[0] * vel[0] + C.G[1] * vel[1] + C.G[2] * vel[2]);
        C.active = true;
    }
    return C;
}

// ------------------------------------------------------------------------------------------------
// Thread-per-point pieces used by the batched path of k_outer (32 points per warp at a time): the parts of the
// per-point work that have no intra-point parallelism worth a warp are run one point per LANE, literally as the
// reference's loops, and only gradientDescent (29-way speculative) stays one point per WARP.
// ------------------------------------------------------------------------------------------------
// choiceTInit<false>(p, 0.15) (sw_manager.hpp:538-581); layer 1 reads the shared pose table.
//
// Layer 1 (the 0.15 s lattice over the whole trajectory, K1 = 134 samples at D = 20 s) is an arg-min with the rule
// "first strict minimum wins, nothing >= 1e9 wins".  That result is the lexicographic minimum of (f_k, k) over the samples
// with f_k < 1e9, whatever the order of evaluation — so samples that PROVABLY cannot attain the minimum need not be
// evaluated.  The shape functors are distances outside the shape: f_k = sdf(R_k^T (p - x_k)) >= |p - x_k| - rout
// (S.rout: circumradius + margin, checked against the oracle for every shape).  Pass 1 finds the lattice pose nearest to p
// (5 flops per sample) and evaluates it: m; pass 2 walks k upwards and evaluates only samples with
// |p - x_k| <= m + rout, tightening m as it goes.  A skipped sample has f_k > m >= the final minimum.  Typically ~15 of
// the 134 samples survive; bits identical to the full scan (GPU parity tests, strict build).
//
// Layers 2 and 3 read their samples' poses from the pose windows (w2, w3; k_pose_table) when those are built: the window is named by
// the layer-1 winner kb and, for layer 3, the layer-2 sample m2 that set the minimum.  The loop's own t still becomes the seed.
template <int SHAPE, bool XFORM>
__device__ __forceinline__ void thread_choice_t_init(const TrajView &tv, const ShapeParams &S, double px, double py,
                                                     const PoseRec *w2, const PoseRec *w3, double &seed, double &min_dis,
                                                     int &evals) {
    const double INF = __longlong_as_double(0x7ff0000000000000LL);
    const uint32_t row = 8u * (uint32_t)tv.K1pad;
    const int K1 = tv.K1;
    // pass 1: nearest lattice pose (rows are 16-byte aligned and K1pad is even: two samples per load)
    double bd2 = INF;
    int k0 = 0;
    {
        uint32_t ps = tv.spose;
#pragma unroll 1
        for (int k = 0; k < K1; k += 2, ps += 16) {
            double x0, x1, y0, y1;
            lds_v2(ps, x0, x1);
            lds_v2(ps + row, y0, y1);
            const double ax = px - x0, ay = py - y0, bx = px - x1, by = py - y1;
            const double d0 = ax * ax + ay * ay, d1 = bx * bx + by * by;
            if (d0 < bd2) { bd2 = d0; k0 = k; }
            if (k + 1 < K1 && d1 < bd2) { bd2 = d1; k0 = k + 1; }
        }
    }
    // pass 2: the nearest pose first (it = -1), then every sample that can still reach the minimum, k ascending; ties are
    // resolved towards the smaller k, so the visiting order does not matter.  One functor call site.
    min_dis = 1e9;
    int kb = -1, ne = 0;
    double thr2 = INF;  // squared pruning radius: |p - x_k| > min_dis + rout  =>  f_k > min_dis
#pragma unroll 1
    for (int it = -1; it < K1; ++it) {
        const int k = (it < 0) ? k0 : it;
        const uint32_t ps = tv.spose + 8u * (uint32_t)k;
        const double xk = lds_f64(ps), yk = lds_f64(ps + row);
        const double ax = px - xk, ay = py - yk;
        const double d2 = ax * ax + ay * ay;
        if (it >= 0 && (!(d2 <= thr2) || k == k0)) continue;
        double rx, ry;
        rel_from_pose(px, py, xk, yk, lds_f64(ps + 2 * row), lds_f64(ps + 3 * row), rx, ry);
        const double f = dev::shape_sdf<SHAPE, XFORM>(S, rx, ry);
        ++ne;
        if (f < min_dis || (f == min_dis && k < kb)) {
            min_dis = f;
            kb = k;
            const double thr0 = f * S.prune_scale + S.rout, thr = fmax(thr0, S.prune_rmin);  // analytic shapes: f * 1 + rout, max with 0
            thr2 = (thr0 >= 0.0) ? thr * thr : INF;      // < 0 cannot happen for a distance function; then no pruning
        }
    }
    seed = (kb >= 0) ? lds_f64(tv.slat + 8u * (uint32_t)kb) : 0.0;
    evals += ne;
    double dt = 0.15;
    int hint = 0;  // piece of the previous sample (the windows are <= 0.3 s wide)
    const PoseRec *win = w2 ? w2 + kWinLen * (kb + 1) : nullptr;  // this layer's window, null: evaluate the trajectory
    int m2 = -1;
#pragma unroll 1
    for (int layer = 2; layer <= 4; ++layer) {
        dt *= 0.1;
        double t = smaxd(0.0, seed - 10 * dt);
        const double term = smind(tv.D, seed + 10 * dt);
#pragma unroll 1
        for (int m = 0; t <= term; t += dt, ++m) {
            double f;
            if (win) {
                const PoseRec cur = ld_pose(win + m);
                double rx, ry;
                rel_from_pose(px, py, cur.x, cur.y, cur.c, cur.s, rx, ry);
                f = dev::shape_sdf<SHAPE, XFORM>(S, rx, ry);
            } else {
                f = eval_sdf<SHAPE, XFORM>(tv, S, px, py, t, hint);
            }
            ++evals;
            if (f < min_dis) {
                seed = t;
                min_dis = f;
                if (layer == 2) m2 = m;
            }
        }
        win = (layer == 2 && w3) ? w3 + kWinLen * (kWin3Stride * (kb + 1) + m2 + 1) : nullptr;
    }
}

// getGradPrelAtTimeStamp (sw_manager.hpp:779-795) -> getonlyGrad1 (Shape.hpp:35-53), one point per thread
template <int SHAPE, bool XFORM, bool SCALED = false>
__device__ __forceinline__ void thread_grad_prel(const TrajView &tv, const ShapeParams &S, double px, double py, double t,
                                                 double &gx, double &gy, const ScaleSched *Z = nullptr) {
    double x, y, yaw, sy, cy, rx, ry;
    traj_pos(tv, t, x, y, yaw);
    dev::sincos_portable(yaw, sy, cy);
    rel_at<SCALED>(Z, t, px, py, x, y, cy, sy, rx, ry);
    if (SHAPE == SH_POLYGON) {
        dev::PolyHit H = dev::polygon_scan(S, rx, ry);
        double vx = rx - H.cx, vy = ry - H.cy;
        double z = vx * vx + vy * vy;
        if (z > 0.0) {
            double n = sqrt(z);
            vx /= n; vy /= n;
        }
        if (H.rs % 2 != 0) { vx = -vx; vy = -vy; }
        gx = vx; gy = vy;
        return;
    }
    if (SHAPE == SH_CIRCLE) {
        dev::circle_grad1<XFORM>(S, rx, ry, gx, gy);
        return;
    }
    const double dx = 0.000001;
    double f[4];
#pragma unroll 1
    for (int q = 0; q < 4; ++q) {  // (x-dx), (x-dx)+2dx, (y-dx), (y-dx)+2dx — one evaluation site
        double qx = rx, qy = ry;
        if (q < 2) { qx -= dx; if (q == 1) qx += 2 * dx; }
        else { qy -= dx; if (q == 3) qy += 2 * dx; }
        f[q] = dev::shape_sdf<SHAPE, XFORM>(S, qx, qy);
    }
    gx = (f[1] - f[0]) / (2 * dx);
    gy = (f[3] - f[2]) / (2 * dx);
}

// ------------------------------------------------------------------------------------------------
// gradientDescent (sw_manager.hpp:1249-1325) for a BATCH of points, a group of 4 lanes per point, each lane evaluating two
// samples per round (8 points in flight per warp) — the batched path of k_outer.
//
// The reference's loop, per descent step: slope sign from the finite difference at x (2 evaluations, recomputed for every
// halving in the reference but always at the same x, hence the same bits), then candidates x - sign * 0.01 * 2^-j for
// j = 0, 1, ... until the first one that decreases f (29 failures end the descent).  Measured on configs 1-3 (oracle,
// orc_descent_stats): ~8 steps per point, accepted j spread evenly over 7..20 (never 1..6), so a full warp per step
// (29 candidates + slope) spends most of its lanes on candidates beyond the accepted one, and one lane per point
// (sequential, 155 +- 65 evaluations) leaves the warp waiting for its slowest lane.  A group runs rounds of 8 samples,
// lane q of the group evaluating samples s = q (slot A) and s = q + 4 (slot B):
//   R1   samples 0/1: the two finite-difference samples; samples 2..7: candidates j = 0..5 in the PREDICTED direction (the
//        slope flips after every non-full step because the accepted step is the largest decreasing one)
//   RN   candidates j = jbase .. jbase + 7 in the known direction (jbase = 6, 14, 22 after R1; 0, 8, 16, 24 after a
//        misprediction)
//   F0   f(x0) when choiceTInit found nothing below 1e9 (degenerate input; the reference evaluates it at iter == 0), and
//        always for a deformable robot (f(x0) of the scaled shape)
// => ~21 sample evaluations per step instead of 31.  The two evaluations of a lane are independent instruction streams
// (latency hiding inside the thread, on top of the resident warps) and the per-round bookkeeping is paid once per two
// evaluations.  Every decision is the sequential loop's decision given the same SDF values: the accepted halving is the
// FIRST j whose candidate decreases f, the sign comes from the finite difference — bit-identical results (GPU parity tests,
// strict build).
// The queue of prepared points is shared by the CTA's 8 warps and holds `limit` / 256 batches of each (wk: chunks of 8 x 32
// entries of 4 doubles: px, py, choiceTInit seed and minimum; entry (c, w, i) at wk[4 (256 c + 32 w + i)], valid for
// i < nbw[8 c + w]; served chunk by chunk, in a chunk i-major, w-minor, through the shared cursor): a group that finishes its
// point writes (sdf, t*) over the entry's seed and minimum and takes the next point of the whole CTA, so the warps of a CTA
// finish together whatever the lengths of their own descents, and the groups idle once per pass, when the queue is empty
// and the longest descent still runs.  Which group solves a point does not change its result; the reductions stay per
// warp, fixed order.
// ------------------------------------------------------------------------------------------------
template <int SHAPE, bool XFORM, bool SCALED = false>
__device__ __forceinline__ void descent_engine2(const TrajView &tv, const ShapeParams &S, double *wk, const int *nbw, int *cursor,
                                                int limit, unsigned &evals SVSDF_STATS_PARAM(unsigned &issued), const ScaleSched *Z = nullptr) {
    enum { E_F0 = 0, E_R1 = 1, E_RN = 2 };
    const int lane = threadIdx.x & 31, q = lane & 3, gbase = lane & 28;
    const double D = tv.D;
    const double INF = __longlong_as_double(0x7ff0000000000000LL);
    const int hi001 = __double2hiint(0.01), lo001 = __double2loint(0.01);
    int pt = -1, mode = E_R1, iter = 0, pred = 1, sgn = 1, jbase = 0, hintA = 0, hintB = 0;
    double px = 0.0, py = 0.0, x = 0.0, fx = 0.0, prev_x = 0.0, t_min = 0.0, t_max = 0.0;
    bool need = true;
#pragma unroll 1
    for (;;) {
        const unsigned want = __ballot_sync(FULL, need && q == 0);
        if (want) {
            int base = 0;
            if (lane == 0) base = atomicAdd(cursor, __popc(want));
            base = __shfl_sync(FULL, base, 0);
            const int c = base + __popc(want & ((1u << gbase) - 1u));
            if (need) {
                pt = -1;
                const int cc = c >> 8, cw = c & (kWarpsPerBlock - 1), ci = (c >> 3) & 31;  // entry (chunk cc, warp cw, point ci)
                need = c < limit;                                          // a hole (ci >= nbw[8 cc + cw]): ask again
                if (c < limit && ci < nbw[kWarpsPerBlock * cc + cw]) {
                    need = false;
                    pt = 256 * cc + 32 * cw + ci;
                    const double *w = wk + 4 * pt;
                    px = w[0]; py = w[1];
                    const double nsd = w[2], nmn = w[3];
                    x = nsd; fx = nmn; prev_x = nsd;   // `prev_x = x` after the (true) first loop test
                    t_min = smaxd(0.0, nsd - 3.4);
                    t_max = smind(nsd + 3.4, D);
                    iter = 0; pred = 1; sgn = 1; jbase = 0; hintA = 0; hintB = 0;
                    mode = (SCALED || nmn >= 1e9) ? E_F0 : E_R1;  // SCALED: f(x0) of the scaled shape
                }
            }
        }
        if (!__any_sync(FULL, pt >= 0)) {
            if (__any_sync(FULL, need)) continue;   // drew only holes: ask again (the queue is not exhausted yet)
            break;
        }

        const bool isR1 = mode == E_R1, isF0 = mode == E_F0;
        const int dir = isR1 ? pred : sgn;
        const int sbit = (dir > 0) ? (int)0x80000000 : 0;
        // slot A: sample s = q (R1: s = 0, 1 are the slope samples, s = 2, 3 candidates j = 0, 1); slot B: s = q + 4
        const bool slopeA = isR1 && q < 2;
        const int jA = isR1 ? q - 2 : jbase + q;
        const int jB = isR1 ? q + 2 : jbase + q + 4;
        const bool candA = !isF0 && !slopeA && jA <= 28, candB = !isF0 && jB <= 28;
        evals += (pt >= 0) ? ((candA || slopeA || (isF0 && q == 0)) ? 1u : 0u) + (candB ? 1u : 0u) : 0u;
        const double offA = slopeA ? ((q == 0) ? -0.000001 : 0.000001) : __hiloint2double((hi001 - ((jA & 31) << 20)) ^ sbit, lo001);
        const double offB = __hiloint2double((hi001 - ((jB & 31) << 20)) ^ sbit, lo001);
        const double loA = slopeA ? ((q == 0) ? 0.0 : -INF) : t_min, hiA = slopeA ? ((q == 0) ? INF : D) : t_max;
        const double tcA = smaxd(smind(x + offA, hiA), loA), tcB = smaxd(smind(x + offB, t_max), t_min);
        const double tA = (candA || slopeA) ? tcA : x, tB = candB ? tcB : x;
        SVSDF_STATS(issued += 64u;)
        const double fA = eval_sdf<SHAPE, XFORM, SCALED>(tv, S, px, py, tA, hintA, Z);
        const double fB = eval_sdf<SHAPE, XFORM, SCALED>(tv, S, px, py, tB, hintB, Z);

        const unsigned balA = __ballot_sync(FULL, (fA - fx) < 0), balB = __ballot_sync(FULL, (fB - fx) < 0);
        const unsigned m8 = ((balA >> gbase) & 0xfu) | (((balB >> gbase) & 0xfu) << 4);
        const double f0 = __shfl_sync(FULL, fA, gbase), f1 = __shfl_sync(FULL, fA, gbase + 1);
        const double g = (f1 - f0) * 500000;
        const int s_new = (int)(g > 0) - (int)(g < 0);
        sgn = isR1 ? s_new : sgn;
        const bool zero = isR1 && sgn == 0;
        const bool mispred = isR1 && sgn != 0 && sgn != pred;
        const int nvalid = max(0, min(8, 29 - jbase));
        const unsigned mc = isR1 ? (m8 >> 2) : (m8 & ((1u << nvalid) - 1u));
        const bool hit = (pt >= 0) && !isF0 && !zero && !mispred && mc != 0u;
        const int k = __ffs(mc) - 1;
        const int jacc = isR1 ? k : jbase + k;
        const int sidx = isR1 ? k + 2 : k;                       // accepted sample index within the round
        const int src = hit ? gbase + (sidx & 3) : lane;
        const bool fromB = (sidx & 4) != 0;
        const double tsel = fromB ? tB : tA, fsel = fromB ? fB : fA;
        const double xacc = __shfl_sync(FULL, tsel, src), facc = __shfl_sync(FULL, fsel, src);
        const int jb_next = isR1 ? (mispred ? 0 : 6) : jbase + 8;
        const bool failed = (pt >= 0) && !isF0 && (zero || (!hit && !mispred && jb_next > 28));
        const bool walking = (jacc == 0) && (xacc == x + (-0.01 * (double)sgn));
        pred = hit ? (walking ? sgn : -sgn) : pred;
        iter += hit ? jacc + 1 : (failed ? 29 : 0);
        x = hit ? xacc : x;
        fx = hit ? facc : (isF0 ? f0 : fx);
        const bool step_end = hit || failed;
        const bool running = (iter < 1000) && !failed && (fabs(x - prev_x) > 1e-16);
        prev_x = step_end ? x : prev_x;
        mode = (step_end || isF0) ? E_R1 : E_RN;
        jbase = jb_next;
        if (step_end && !running) {
            if (q == 0) { wk[4 * pt + 2] = fx; wk[4 * pt + 3] = x; }
            pt = -1;
            need = true;
        }
    }
    __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// TMA bulk copy of the trajectory blob into shared memory (cp.async.bulk + mbarrier)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void tma_load_blob(double *smem_blob, const double *gmem_blob, int n_doubles,
                                              uint64_t *bar) {
    const uint32_t bar_a = smem_u32(bar);
    const uint32_t bytes = (uint32_t)n_doubles * 8u;
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar_a), "r"(1));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                smem_u32(smem_blob)),
            "l"(gmem_blob), "r"(bytes), "r"(bar_a)
            : "memory");
    }
    // all threads wait on phase 0
    uint32_t done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar_a), "r"(0)
            : "memory");
    }
}

// ------------------------------------------------------------------------------------------------
// k_pose_table: (x, y, cos yaw, sin yaw) at the layer-1 lattice times, written into the blob in place.
// The lattice and its poses are shared by every query point (choiceTInit layer 1 always scans 0..D in 0.15 s
// steps), so they are computed once per evaluation instead of once per point.  Rigid for a deformable robot too: the
// layer-1 scan does not read the scale.
// ------------------------------------------------------------------------------------------------
// (shared with k_pose_table_multi, svsdf_kernels_multi.cuh)
__device__ __forceinline__ void pose_table_entry(double *blob, int k) {
    TrajView tv = make_view(blob);
    if (k >= tv.K1) return;
    double x, y, yaw, sy, cy;
    traj_pos(tv, tv.lat[k], x, y, yaw);
    dev::sincos_portable(yaw, sy, cy);
    const BlobLayout L = blob_layout(tv.N, tv.K1);
    double *ps = blob + L.off_pose + k;
    ps[0] = x; ps[L.K1pad] = y; ps[2 * L.K1pad] = cy; ps[3 * L.K1pad] = sy;
}
// Record e of the pose windows of choiceTInit layers 2 (e < win2_records) and 3 (the rest; w3 null: none), svsdf_types.h:PoseRec.
// The thread replays the scan loops' arithmetic on the window's seed: dt *= 0.1 per layer, the clamped start smaxd(0, seed - 10 dt),
// then t += dt once per earlier sample (for layer 3 first the layer-2 chain up to sample m2, which is the seed) — the same operations
// on the same bits, so the pose is the one eval_sdf computes at the loop's t.  Rigid: the seed layers never read the scale.
__device__ __forceinline__ void pose_window_entry(const double *blob, PoseRec *w2, PoseRec *w3, int64_t e) {
    const TrajView tv = make_view(blob);
    const int64_t n2 = win2_records(tv.K1);
    const bool layer3 = e >= n2;
    if (layer3) {
        e -= n2;
        if (!w3 || e >= win3_records(tv.K1)) return;
    }
    PoseRec *out = (layer3 ? w3 : w2) + e;
    const int64_t w = e / kWinLen;
    const int m = (int)(e - w * kWinLen);
    const int kb = (int)(layer3 ? w / kWin3Stride : w) - 1;
    const int m2 = layer3 ? (int)(w % kWin3Stride) - 1 : -1;
    double seed = (kb >= 0) ? tv.lat[kb] : 0.0;
    double dt = 0.15;
    dt *= 0.1;
    if (m2 >= 0) {
        double t = smaxd(0.0, seed - 10 * dt);
        for (int i = 0; i < m2; ++i) t += dt;
        seed = t;
    }
    if (layer3) dt *= 0.1;
    double t = smaxd(0.0, seed - 10 * dt);
    for (int i = 0; i < m; ++i) t += dt;
    double x, y, yaw, sy, cy;
    traj_pos(tv, t, x, y, yaw);
    dev::sincos_portable(yaw, sy, cy);
    out->x = x; out->y = y; out->c = cy; out->s = sy;
}

// ------------------------------------------------------------------------------------------------
// K1: outer solve for every point (+ penalty, chain rule and CTA reduction for outside points)
// dynamic smem: [ blob | 8 warps x (19N + 1) accumulators ]
// ------------------------------------------------------------------------------------------------
#ifndef SVSDF_MESH_MIN_CTAS
#define SVSDF_MESH_MIN_CTAS 4  // measured on config 4m: 2 -> 245 ms, 3 -> 206 ms, 4 -> 198 ms (the traversal is latency bound; spills stay in L1)
#endif
#ifndef SVSDF_OUTER_MIN_CTAS
#define SVSDF_OUTER_MIN_CTAS 3
#endif
#ifndef SVSDF_GSIP_MIN_CTAS
#define SVSDF_GSIP_MIN_CTAS 3
#endif
// BATCHED selects the schedule at compile time (two kernels: each carries only its own evaluation sites).
// SCALED: deformable robot with the schedule *Z (k_outer_scaled); the rigid k_outer passes nullptr and never reads it.
// vblock / vgrid: this CTA's index and the grid it belongs to — blockIdx.x / gridDim.x for k_outer; for k_outer_multi the
// problem's virtual grid, so that every problem keeps the decomposition (and the partial sums) of its single-problem call.
template <int SHAPE, bool XFORM, bool BATCHED, bool SCALED>
__device__ __forceinline__ void outer_body(const KernelArgs &A, const ShapeParams &S, const ScaleSched *Z, int vblock, int vgrid) {
    extern __shared__ __align__(16) double smem[];
    __shared__ __align__(8) uint64_t bar;
    __shared__ int s_nb[kOuterChunkMax * kWarpsPerBlock];
    __shared__ int s_cursor;
    double *sblob = smem;
    tma_load_blob(sblob, A.blob, A.blob_doubles, &bar);
    const TrajView tv = make_view(sblob);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nacc = 19 * tv.N + 1;
    double *acc = smem + A.blob_doubles + warp * nacc;  // [N][18] gdC, then [N] gdT-by-piece, then cost
    if (A.want_reduce)
        for (int e = lane; e < nacc; e += 32) acc[e] = 0.0;
    __syncwarp();

    const int64_t wstride = (int64_t)vgrid * kWarpsPerBlock;
    const int64_t first = (int64_t)vblock * kWarpsPerBlock + warp;
    unsigned long long my_evals = 0;
    double *res = smem + A.blob_doubles + kWarpsPerBlock * nacc + warp * 128;  // per-warp work area of the descent engine
    // The warp walks its points in batches of up to 32 (lane i <-> i-th point of the batch).
    //  * Batched schedule (large P): the points are cut into nB = W * ceil(P / 32 W) CONTIGUOUS batches of equal size
    //    (+-1; neighbouring map cells: the lanes of a warp then prune the same layer-1 samples and run descents of similar
    //    length), warp w owns batches w, w + W, ... (strided: a warp's batches come from different regions of the map, so
    //    hard regions are spread over the warps; static, hence deterministic).  choiceTInit and the FD gradient /
    //    penalty / chain rule run one point per lane, gradientDescent one point per group of 4 lanes, served from the CTA's
    //    point queue (descent_engine2).  A pass takes up to A.outer_chunk batches of every warp: their seeds go into the queue
    //    batch after batch, ONE descent pass drains it, then the warp finishes its batches in order.  The descents' lengths
    //    vary by +-40 %, so every pass ends with groups idling until the longest one is done: fewer, longer passes idle less.
    //    Nothing but the work area lives across the descent; the epilogue reads the point back from it.
    //  * Sparse schedule (few points per warp, i.e. small problems): the warp owns points w, w + W, ...; everything one
    //    point per warp, as solve_outer / grad_prel do (lowest latency).
    const int64_t lstride = BATCHED ? 1 : wstride;  // distance between the points of neighbouring lanes
    const int64_t nB = wstride * ((A.P + 32 * wstride - 1) / (32 * wstride));   // batches (batched schedule)
    const int chunk = BATCHED ? A.outer_chunk : 1;  // batches of a warp per descent pass
    SVSDF_STATS(unsigned long long st_issued = 0, st_useful = 0, st_seed = 0, st_desc = 0, st_wait = 0, st_epi = 0;)
    for (int64_t bi = first; BATCHED ? (bi < nB) : (bi < A.P); bi += BATCHED ? chunk * wstride : 32 * wstride) {
        int nc = 1;  // batches of this pass: bi, bi + W, ...  (nB is a multiple of W: the same for every warp of the CTA)
        if (BATCHED) {  // the whole CTA: the batched schedule synchronises the CTA around its shared queue
            nc = (int)min((int64_t)chunk, (nB - bi + wstride - 1) / wstride);
            SVSDF_STATS(const long long c0 = clock64();)
            int ev = 0;
#pragma unroll 1
            for (int c = 0; c < nc; ++c) {  // seeds of batch c, one point per lane, into work-area entry (c, warp, lane)
                const int64_t b = bi + c * wstride;
                const int64_t bfirst = (b * A.P) / nB;
                const int nb = (int)min((int64_t)32, ((b + 1) * A.P) / nB - bfirst);
                if (lane < nb) {
                    const double px = __ldg(A.points_xy + 2 * (bfirst + lane)), py = __ldg(A.points_xy + 2 * (bfirst + lane) + 1);
                    double seed = 0.0, mn = 1e9;
                    thread_choice_t_init<SHAPE, XFORM>(tv, S, px, py, A.win2, A.win3, seed, mn, ev);
                    double *e = res + 1024 * c + 4 * lane;
                    e[0] = px; e[1] = py; e[2] = seed; e[3] = mn;
                }
                __syncwarp();
                if (lane == 0) s_nb[kWarpsPerBlock * c + warp] = nb;
            }
            unsigned ev2 = 0;
            SVSDF_STATS(unsigned issued = 0;)
            if (threadIdx.x == 0) s_cursor = 0;
            SVSDF_STATS(const long long c1 = clock64();)
            __syncthreads();
            SVSDF_STATS(const long long c2 = clock64();)
            descent_engine2<SHAPE, XFORM, SCALED>(tv, S, res - 128 * warp, s_nb, &s_cursor, nc * kWarpsPerBlock * 32, ev2 SVSDF_STATS_PARAM(issued), Z);
            SVSDF_STATS(const long long c3 = clock64();)
            __syncthreads();
            SVSDF_STATS(const long long c4 = clock64(); st_seed += c2 - c0; st_desc += c3 - c2; st_wait += c4 - c3;
                        st_issued += issued; st_useful += __reduce_add_sync(FULL, ev2);)
            my_evals += (unsigned long long)__reduce_add_sync(FULL, (unsigned)ev + ev2);
            __syncwarp();
        }
        SVSDF_STATS(const long long c5 = clock64();)
#pragma unroll 1
        for (int c = 0; c < nc; ++c) {  // the batches of the pass in their own order: the warp's summation chain (sparse: one)
            // batched: batch b covers [b P / nB, (b + 1) P / nB); sparse: points bi, bi + W, ...
            const int64_t b = bi + c * wstride;
            const int64_t bfirst = BATCHED ? (b * A.P) / nB : b;
            const int64_t bend = BATCHED ? ((b + 1) * A.P) / nB : A.P;
            const int64_t my_pt = bfirst + (int64_t)lane * lstride;
            const int nb = (int)min((int64_t)32, (bend - bfirst + lstride - 1) / lstride);  // batch size (warp-uniform)
            const bool my_valid = lane < nb;
            double mpx = 0.0, mpy = 0.0, m_sdf = 0.0, m_ts = 0.0, m_gx = 0.0, m_gy = 0.0;
            if (BATCHED) {
                const double *e = res + 1024 * c + 4 * lane;
                if (my_valid) { mpx = e[0]; mpy = e[1]; m_sdf = e[2]; m_ts = e[3]; }
            } else {
                const int64_t ld_pt = my_valid ? my_pt : bfirst;
                mpx = __ldg(A.points_xy + 2 * ld_pt); mpy = __ldg(A.points_xy + 2 * ld_pt + 1);
#pragma unroll 1
                for (int i = 0; i < nb; ++i) {
                    const double px = __shfl_sync(FULL, mpx, i), py = __shfl_sync(FULL, mpy, i);
                    const OuterResult R = solve_outer<SHAPE, XFORM, SCALED>(tv, S, px, py, A.win2, A.win3, false, 0.0, 1e9, Z);
                    my_evals += (unsigned long long)R.evals;
                    if (lane == i) { m_sdf = R.sdf; m_ts = R.tstar; }
                    double gx, gy;
                    grad_prel<SHAPE, XFORM, SCALED>(tv, S, px, py, R.tstar, gx, gy, Z);
                    if (lane == i) { m_gx = gx; m_gy = gy; }
                }
            }
            my_evals += 4ull * (unsigned long long)nb;
            if (BATCHED && my_valid) thread_grad_prel<SHAPE, XFORM, SCALED>(tv, S, mpx, mpy, m_ts, m_gx, m_gy, Z);
            // ---- per-lane epilogue: outputs, interior flag, penalty + chain rule (one point per lane) ----
            const bool inside = my_valid && A.want_gsip && !(m_sdf > 0);  // getTrueSDFofSweptVolume: `if (argmin_dis > 0) return`
            if (my_valid) {
                if (A.out_sdf) A.out_sdf[my_pt] = m_sdf;
                if (A.out_tstar) A.out_tstar[my_pt] = m_ts;
                if (A.out_grad) { A.out_grad[3 * my_pt] = m_gx; A.out_grad[3 * my_pt + 1] = m_gy; A.out_grad[3 * my_pt + 2] = 0.0; }
                if (A.out_rounds) A.out_rounds[my_pt] = 0;
                if (A.inside_flag) A.inside_flag[my_pt] = inside ? 1 : 0;
                if (inside && A.inside_tstar) A.inside_tstar[my_pt] = m_ts;
            }
            if (A.want_reduce) {
                Contribution C;
                C.active = false;
                if (my_valid && !inside) C = point_contribution<SCALED>(tv, A.cp, mpx, mpy, m_sdf, m_ts, m_gx, m_gy, Z);
                // accumulate the active lanes' contributions in batch order (deterministic)
                unsigned m = __ballot_sync(FULL, C.active);
                while (m) {
                    const int src = __ffs(m) - 1;
                    m &= m - 1;
                    const int piece = __shfl_sync(FULL, C.piece, src);
                    const double s1 = __shfl_sync(FULL, C.s1, src);
                    const double g0 = __shfl_sync(FULL, C.G[0], src), g1 = __shfl_sync(FULL, C.G[1], src),
                                 g2 = __shfl_sync(FULL, C.G[2], src);
                    const double gdT = __shfl_sync(FULL, C.gdT, src), pena = __shfl_sync(FULL, C.pena, src);
                    if (lane < 18) {
                        const int d = lane / 6, q = lane - 6 * d;
                        const double s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2, s5 = s4 * s1;
                        const double beta = (q == 0) ? 1.0 : (q == 1) ? s1 : (q == 2) ? s2 : (q == 3) ? s3 : (q == 4) ? s4 : s5;
                        const double gd = (d == 0) ? g0 : (d == 1) ? g1 : g2;
                        acc[piece * 18 + lane] += beta * gd;
                    } else if (lane == 18) {
                        acc[18 * tv.N + piece] += gdT;
                    } else if (lane == 19) {
                        acc[19 * tv.N] += pena;
                    }
                    __syncwarp();
                }
            }
        }
        SVSDF_STATS(if (BATCHED) st_epi += clock64() - c5;)
    }
    SVSDF_STATS(if (BATCHED && g_phase_stats && lane == 0) {
        unsigned long long *st = g_phase_stats + 6 * ((size_t)blockIdx.x * kWarpsPerBlock + warp);
        st[0] = st_issued; st[1] = st_useful; st[2] = st_seed; st[3] = st_desc; st[4] = st_wait; st[5] = st_epi;
    })
    if (A.eval_counter && lane == 0) atomicAdd(A.eval_counter, my_evals);
    if (A.want_reduce) {
        __syncthreads();
        const double *acc0 = smem + A.blob_doubles;
        for (int e = threadIdx.x; e < nacc; e += blockDim.x) {
            double s = 0.0;
#pragma unroll
            for (int w = 0; w < kWarpsPerBlock; ++w) s += acc0[w * nacc + e];
            A.partials[(int64_t)vblock * nacc + e] = s;
        }
    }
}
template <int SHAPE, bool XFORM, bool BATCHED>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, (SHAPE == SH_MESH) ? SVSDF_MESH_MIN_CTAS : SVSDF_OUTER_MIN_CTAS)
    k_outer(const __grid_constant__ KernelArgs A, const __grid_constant__ ShapeParams S) {
    outer_body<SHAPE, XFORM, BATCHED, false>(A, S, nullptr, blockIdx.x, gridDim.x);
}
template <int SHAPE, bool XFORM, bool BATCHED>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, (SHAPE == SH_MESH) ? SVSDF_MESH_MIN_CTAS : SVSDF_OUTER_MIN_CTAS)
    k_outer_scaled(const __grid_constant__ KernelArgs A, const __grid_constant__ ShapeParams S, const __grid_constant__ ScaleSched Z) {
    outer_body<SHAPE, XFORM, BATCHED, true>(A, S, &Z, blockIdx.x, gridDim.x);
}

// ------------------------------------------------------------------------------------------------
// k_compact: ordered compaction of the inside flags (single CTA, 1024 threads) -> inside_list, n_inside.
// Flags are 0/1 bytes; every thread owns a contiguous run of 16-byte words (coalesced uint4 loads, popcount).
// ------------------------------------------------------------------------------------------------
// (the body is shared with k_compact_multi, one CTA per problem; flag must be 16-byte aligned)
__device__ __forceinline__ void compact_body(const unsigned char *flag, int64_t P, int *list, int *n_out) {
    __shared__ int wsum[32];
    __shared__ int total;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t nwords = (P + 15) / 16;              // flag buffer is allocated with >= 16 bytes of slack
    const int64_t per = (nwords + 1023) / 1024;        // words per thread
    const int64_t w0 = (int64_t)tid * per, w1 = (w0 + per < nwords) ? w0 + per : nwords;
    const uint4 *f4 = reinterpret_cast<const uint4 *>(flag);
    int cnt = 0;
    for (int64_t w = w0; w < w1; ++w) {
        uint4 v = f4[w];
        if (16 * w + 16 > P) {  // mask the tail beyond P
            unsigned char *b = reinterpret_cast<unsigned char *>(&v);
            for (int q = 0; q < 16; ++q)
                if (16 * w + q >= P) b[q] = 0;
        }
        cnt += __popc(v.x) + __popc(v.y) + __popc(v.z) + __popc(v.w);
    }
    int inc = cnt;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        int v = __shfl_up_sync(FULL, inc, off);
        if (lane >= off) inc += v;
    }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        int v = wsum[lane];
        int vi = v;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            int u = __shfl_up_sync(FULL, vi, off);
            if (lane >= off) vi += u;
        }
        wsum[lane] = vi - v;  // exclusive
        if (lane == 31) total = vi;
    }
    __syncthreads();
    int pos = wsum[warp] + inc - cnt;
    if (cnt > 0) {
        for (int64_t w = w0; w < w1; ++w) {
            const uint4 v = f4[w];
            if ((v.x | v.y | v.z | v.w) == 0u) continue;
            const unsigned char *b = reinterpret_cast<const unsigned char *>(&v);
            for (int q = 0; q < 16; ++q) {
                const int64_t i = 16 * w + q;
                if (i < P && b[q]) list[pos++] = (int)i;
            }
        }
    }
    if (tid == 0) *n_out = total;
}

// ------------------------------------------------------------------------------------------------
// K2: interior branch of getTrueSDFofSweptVolume<true> (sw_manager.hpp:926-1017, SampleSet2D :41-124).
// One CTA per inside point; the ring samples of a round are distributed over the CTA's warps, each warp
// running a full outer solve on its sample.
// dynamic smem: [ blob ]
// ------------------------------------------------------------------------------------------------
// SCALED: the ring samples run scaled descents (getSDFofSweptVolume<useScale>); the velocity fallback and the ring do not change.
// The slots of the interior branch come from a VIEW: GsipSingle below (k_gsip: one blob, loaded once, slot s = inside point
// A.inside_list[s]); k_gsip_multi's view (svsdf_kernels_multi.cuh) maps a slot of the concatenated lists to its problem and reloads the
// CTA's blob when the problem changes.  The body is the same for both.
struct GsipSingle {
    const KernelArgs &A;
    __device__ __forceinline__ void start(double *sblob, uint64_t *bar) const { tma_load_blob(sblob, A.blob, A.blob_doubles, bar); }
    __device__ __forceinline__ int count() const { return *A.n_inside; }
    // point index of the slot and the arrays it indexes; true when the blob in shared memory was replaced (never here)
    __device__ __forceinline__ bool at(int slot, double *, uint64_t *, int &pt, const double *&pts, const double *&tstar) const {
        pt = A.inside_list[slot];
        pts = A.points_xy;
        tstar = A.inside_tstar;
        return false;
    }
};
template <int SHAPE, bool XFORM, int WARPS, bool SCALED, class View>
__device__ __forceinline__ void gsip_body(const KernelArgs &A, const ShapeParams &S, const ScaleSched *Z, const View &view) {
    extern __shared__ __align__(16) double smem[];
    __shared__ __align__(8) uint64_t bar;
    __shared__ double s_theta[24], s_val[24], s_ts[24];
    double *sblob = smem;
    view.start(sblob, &bar);
    TrajView tv = make_view(sblob);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double PI = 3.14159265358979323846;  // Shape.hpp:31
    const int n_in = view.count();
    unsigned long long my_evals = 0;

    for (int slot = blockIdx.x; slot < n_in; slot += gridDim.x) {
        int pt;
        const double *pts, *in_tstar;
        if (view.at(slot, sblob, &bar, pt, pts, in_tstar)) tv = make_view(sblob);
        const double px = __ldg(pts + 2 * (int64_t)pt), py = __ldg(pts + 2 * (int64_t)pt + 1);
        const double ts0 = in_tstar[pt];
        // velocity at t* with the reference's fallback scan (:928-954); all threads redundantly
        double vx, vy, vw;
        traj_vel(tv, ts0, vx, vy, vw);
        if (sqrt(vx * vx + vy * vy + vw * vw) < 0.01) {
            if (ts0 < 0.1) {
                for (double t_scan = ts0; t_scan <= tv.D; t_scan += 0.1) {
                    traj_vel(tv, t_scan, vx, vy, vw);
                    if (sqrt(vx * vx + vy * vy + vw * vw) >= 0.01) break;
                }
            } else if (ts0 > tv.D - 0.1) {
                for (double t_scan = ts0; t_scan >= 0; t_scan -= 0.1) {
                    traj_vel(tv, t_scan, vx, vy, vw);
                    if (sqrt(vx * vx + vy * vy + vw * vw) >= 0.01) break;
                }
            }
        }
        // SampleSet2D::initSet (:74-103)
        double r = 10.0;
        double theta0 = dev::atan2_portable(vx, -vy);
        if (theta0 < 0) theta0 += 2 * PI;
        double theta_res = PI + 0.1;
        double r_star = 0.0, real_t_star = 0.0, star_theta = 0.0;
        int iter = 1, rounds = 0;
        while (true) {
            // getElements (:59-71): one ring (rk = 1.0), theta accumulated from theta0 while < theta0 + 2 PI
            int ns = 0;
            for (double th = theta0; th < theta0 + 2 * PI; th += theta_res) {
                if (threadIdx.x == 0 && ns < 24) s_theta[ns] = th;
                ns++;
            }
            if (ns > 24) ns = 24;  // cannot happen: theta_res >= 0.3 -> at most 21 samples
            __syncthreads();
            for (int k = warp; k < ns; k += WARPS) {
                double th = s_theta[k];
                double sn, cs;
                dev::sincos_portable(th, sn, cs);
                double yx = px + 1.0 * r * cs, yy = py + 1.0 * r * sn;  // CircleCoord2D::getPosition (:36-39)
                OuterResult R = solve_outer<SHAPE, XFORM, SCALED>(tv, S, yx, yy, A.win2, A.win3, false, 0.0, 1e9, Z);
                my_evals += (unsigned long long)R.evals;
                if (lane == 0) { s_val[k] = R.sdf; s_ts[k] = R.tstar; }
            }
            __syncthreads();
            double max_g = -100000;
            for (int k = 0; k < ns; ++k) {
                double cur = s_val[k];
                if (cur > max_g) {
                    max_g = cur;
                    real_t_star = s_ts[k];
                    star_theta = s_theta[k];
                }
            }
            __syncthreads();  // everyone has read s_* before the next round overwrites them
            r_star = r - max_g;
            r = r_star;
            rounds++;
            if (iter > 8) break;
            if (fabs(max_g) < 0.1) break;
            theta_res /= (2 + 1);  // expandSet(2, theta*) (:105-123)
            theta_res = smaxd(0.3, theta_res);
            theta0 = star_theta;
            iter++;
        }
        double sn, cs;
        dev::sincos_portable(star_theta, sn, cs);
        double corx = px + 1.0 * r_star * cs, cory = py + 1.0 * r_star * sn;
        double gx = corx - px, gy = cory - py;
        double z = gx * gx + gy * gy;
        if (z > 0) {
            double n = sqrt(z);
            gx /= n; gy /= n;
        }
        const double sdf = -r_star;
        if (threadIdx.x == 0) {
            if (A.out_sdf) A.out_sdf[pt] = sdf;
            if (A.out_tstar) A.out_tstar[pt] = real_t_star;
            if (A.out_grad) { A.out_grad[3 * pt] = gx; A.out_grad[3 * pt + 1] = gy; A.out_grad[3 * pt + 2] = 0.0; }
            if (A.out_rounds) A.out_rounds[pt] = rounds;
        }
        if (A.want_reduce && warp == 0) {
            Contribution C = point_contribution<SCALED>(tv, A.cp, px, py, sdf, real_t_star, gx, gy, Z);
            double *o = A.gsip_contrib + 20 * (int64_t)slot;
            if (lane < 18) {
                int d = lane / 6, q = lane - 6 * d;
                double s1 = C.s1, s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2, s5 = s4 * s1;
                double beta = (q == 0) ? 1.0 : (q == 1) ? s1 : (q == 2) ? s2 : (q == 3) ? s3 : (q == 4) ? s4 : s5;
                o[1 + lane] = C.active ? beta * C.G[d] : 0.0;
            } else if (lane == 18) {
                o[19] = C.active ? C.gdT : 0.0;
            } else if (lane == 19) {
                o[0] = C.active ? C.pena : 0.0;
                A.gsip_piece[slot] = C.piece;
            }
        }
    }
    if (A.eval_counter && lane == 0) atomicAdd(A.eval_counter, my_evals);
}
template <int SHAPE, bool XFORM, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, (WARPS == kWarpsPerBlock && SHAPE != SH_MESH) ? SVSDF_GSIP_MIN_CTAS : 1)
    k_gsip(const __grid_constant__ KernelArgs A, const __grid_constant__ ShapeParams S) {
    gsip_body<SHAPE, XFORM, WARPS, false>(A, S, nullptr, GsipSingle{A});
}
template <int SHAPE, bool XFORM, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, (WARPS == kWarpsPerBlock && SHAPE != SH_MESH) ? SVSDF_GSIP_MIN_CTAS : 1)
    k_gsip_scaled(const __grid_constant__ KernelArgs A, const __grid_constant__ ShapeParams S, const __grid_constant__ ScaleSched Z) {
    gsip_body<SHAPE, XFORM, WARPS, true>(A, S, &Z, GsipSingle{A});
}

// ------------------------------------------------------------------------------------------------
// k_finalize: fixed-order sum of the K1 CTA partials and the K2 per-point contributions.  One warp per accumulator
// entry: lane l adds partials l, l+32, ... in order, the 32 lane sums are combined by a fixed shuffle tree, so the
// result is bit-reproducible.  The last CTA to finish (ticket counter) writes the output record:
// out: [0] cost, [1 .. 18N] gradC in Eigen column-major order (d*6N + 6i + q), [1+18N .. 1+19N) gradT with the
// reference's rule gradT(j) += gdT for all j < piece (back_end_optimizer.hpp:859-862), [1+19N] n_inside.
// (k_finalize itself, svsdf_kernels_shared.cuh, lives in the rigid units only: the scaled units share it.)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum_fixed(double v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(FULL, v, off);
    return __shfl_sync(FULL, v, 0);
}

// bx / nbx: this CTA's index among the nbx CTAs that finalize one record (blockIdx.x / gridDim.x for k_finalize; k_finalize_multi
// runs one such group per problem)
__device__ __forceinline__ void finalize_body(const double *partials, int n_blocks, int N, int n_in, const double *gsip_contrib,
                                              const int *gsip_piece, double *tot, unsigned int *ticket, double *out, int bx, int nbx) {
    const int nacc = 19 * N + 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int e = bx * 8 + warp;
    if (e < nacc) {
        double s = 0.0;
        for (int b = lane; b < n_blocks; b += 32) s += partials[(int64_t)b * nacc + e];
        s = warp_sum_fixed(s);
        // K2 contributions, ascending point order (inside_list is sorted)
        double s2 = 0.0;
        if (e < 18 * N) {
            const int piece = e / 18, within = e - 18 * piece;
            for (int k = lane; k < n_in; k += 32)
                if (gsip_piece[k] == piece) s2 += gsip_contrib[20 * (int64_t)k + 1 + within];
        } else if (e < 19 * N) {
            const int piece = e - 18 * N;
            for (int k = lane; k < n_in; k += 32)
                if (gsip_piece[k] == piece) s2 += gsip_contrib[20 * (int64_t)k + 19];
        } else {
            for (int k = lane; k < n_in; k += 32) s2 += gsip_contrib[20 * (int64_t)k];
        }
        s2 = warp_sum_fixed(s2);
        if (lane == 0) tot[e] = s + s2;
    }
    __shared__ bool last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = (atomicAdd(ticket, 1u) == (unsigned)nbx - 1);
    __syncthreads();
    if (!last) return;
    __threadfence();
    for (int q = threadIdx.x; q < nacc; q += blockDim.x) {
        if (q < 18 * N) {
            const int piece = q / 18, within = q - 18 * piece;
            const int d = within / 6, pw = within - 6 * d;
            out[1 + d * 6 * N + 6 * piece + pw] = __ldcg(tot + q);
        } else if (q < 19 * N) {
            const int j = q - 18 * N;
            double sfx = 0.0;
            for (int i = j + 1; i < N; ++i) sfx += __ldcg(tot + 18 * N + i);
            out[1 + 18 * N + j] = sfx;
        } else {
            out[0] = __ldcg(tot + q);
        }
    }
    if (threadIdx.x == 0) {
        out[1 + 19 * N] = (double)n_in;
        *ticket = 0u;  // re-arm for the next evaluation
    }
}

// ------------------------------------------------------------------------------------------------
// Host-side helpers of the cost launchers.  A variant's kernel list K (CostKernels, MultiKernels) names its kernels: K::outer(batched),
// the sparse or batched k_outer, and K::gsip(wide), the 8- or 22-warp k_gsip.
// ------------------------------------------------------------------------------------------------
// Opts K's four kernels in to kMaxDynSmemBytes of dynamic shared memory, once per device ordinal: the attribute is per device (a
// process may hold contexts on several GPUs).
template <class K>
static cudaError_t raise_smem_cap() {
    static bool attr_set_dev[64] = {};
    int dev_ord = 0;
    cudaGetDevice(&dev_ord);
    bool &attr_set = attr_set_dev[dev_ord & 63];
    if (attr_set) return cudaSuccess;
    for (const void *k : {(const void *)K::outer(false), (const void *)K::outer(true), (const void *)K::gsip(false), (const void *)K::gsip(true)}) {
        const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmemBytes);
        if (e != cudaSuccess) return e;
    }
    attr_set = true;
    return cudaSuccess;
}

// Launches one of a variant's kernels on args; a deformable robot's (SCALED) take the scale schedule *Z after them.
template <bool SCALED, class Kernel, class... Args>
static cudaError_t launch_cost(Kernel k, int grid, int threads, size_t smem, cudaStream_t st, const ScaleSched *Z, const Args &...args) {
    if constexpr (SCALED) k<<<grid, threads, smem, st>>>(args..., *Z);
    else k<<<grid, threads, smem, st>>>(args...);
    return cudaGetLastError();
}

}  // namespace SVSDF_NS
}  // namespace svsdf
