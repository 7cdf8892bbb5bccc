// svsdf_pose.cu — the pose-sampled obstacle penalty (svsdf_set_pose_penalty): the reference's grad_cost_p
// (back_end_optimizer.hpp:956-1028) at every sample of addTimeIntPenalty (:411-533), for every problem of a call.
//
// One warp per (problem, piece, sample).  The sample's pose x = c_i^T beta0(s) gives the box of voxels the reference gathers
// (PCSmapManager::getPointsInAABB, PCSmap_manager.h:160-182: map_index_box, then i, j, k ascending with k innermost); the warp's lanes
// take 32 consecutive cells of that order at a time, test the map bit and, for an occupied cell whose body-frame offset passes the
// box filter, evaluate the functor and its gradient (getSDFwithGrad1) and the smoothed-L1 terms.  The active cells' terms are then
// summed one after the other in the cells' order, as the reference's loop sums them; every lane holds the sums, lane 0 writes the
// sample's record (costp, gradp_x, gradp_y, grad_yaw).  The loop runs over the whole box in chunks: no cap on the cells per box and
// no buffer sized by it.
//
// Compiled twice: -DSVSDF_NS=fast (FMA contraction) and -DSVSDF_NS=strict -fmad=false (the reference's rounding).  Cell centres are
// ((i + 0.5) res + lo) rounded as the host and the extraction round them in both builds.
#include <cuda_runtime.h>
#include <stdint.h>

#include "host/minco.hpp"
#include "svsdf_launch.h"
#include "svsdf_shapes.cuh"
#include "svsdf_sincos.cuh"
#include "svsdf_types.h"

#ifndef SVSDF_NS
#error "compile svsdf_pose.cu with -DSVSDF_NS=fast or -DSVSDF_NS=strict"
#endif

namespace svsdf {
namespace SVSDF_NS {
namespace {

constexpr int kPoseWarps = 4;
constexpr unsigned kFull = 0xffffffffu;

// getSDFwithGrad1 at the body-frame point (rx, ry): the value and the gradient's x, y (its z is 0 for every functor here).
// Generic shapes: helperfunc (Shape.hpp:53-72), the value then the central differences of getonlyGrad1.  Polygon: its override
// (Shape.hpp:1536-1566), one edge scan for both.  Circle: its override (:497-503), whose value is |p_rel.head(2)| - radius WITHOUT
// the poly_params transform (getonlySDF applies it), and whose gradient is circle_grad1's.
template <int SHAPE, bool XFORM>
__device__ __forceinline__ double sdf_with_grad1(const ShapeParams &S, double rx, double ry, double &gx, double &gy) {
    if (SHAPE == SH_POLYGON) {
        const dev::PolyHit H = dev::polygon_scan(S, rx, ry);
        double vx = rx - H.cx, vy = ry - H.cy;
        const double z = vx * vx + vy * vy;
        if (z > 0.0) {
            const double n = sqrt(z);
            vx /= n; vy /= n;
        }
        if (H.rs % 2 != 0) { vx = -vx; vy = -vy; }
        gx = vx; gy = vy;
        return (H.rs % 2 == 0) ? H.dis : -H.dis;
    }
    if (SHAPE == SH_CIRCLE) {
        dev::circle_grad1<XFORM>(S, rx, ry, gx, gy);
        return dev::shape_sdf<SH_CIRCLE, false>(S, rx, ry);
    }
    const double sdf = dev::shape_sdf<SHAPE, XFORM>(S, rx, ry);
    const double dx = 0.000001;
    double t0 = rx, t1 = ry;
    t0 -= dx;
    double sdfold = dev::shape_sdf<SHAPE, XFORM>(S, t0, t1);
    t0 += 2 * dx;
    const double gradx = dev::shape_sdf<SHAPE, XFORM>(S, t0, t1) - sdfold;
    t0 = rx;
    t1 -= dx;
    sdfold = dev::shape_sdf<SHAPE, XFORM>(S, t0, t1);
    t1 += 2 * dx;
    const double grady = dev::shape_sdf<SHAPE, XFORM>(S, t0, t1) - sdfold;
    gx = gradx / (2 * dx);
    gy = grady / (2 * dx);
    return sdf;
}

template <int SHAPE, bool XFORM>
__global__ void __launch_bounds__(kPoseWarps * 32) k_pose(const PoseArgs A, const __grid_constant__ ShapeParams S) {
    const int lane = threadIdx.x & 31;
    const PoseProblem pr = A.prob ? A.prob[blockIdx.y] : PoseProblem{0, 0};
    const double *blob = A.blobs + pr.blob_off;
    const int N = (int)blob[0], R = A.res_samples;
    const int item = blockIdx.x * kPoseWarps + (int)(threadIdx.x >> 5);
    if (item >= N * (R + 1)) return;
    const int i = item / (R + 1), j = item - i * (R + 1);
    const BlobLayout L = blob_layout(N, (int)blob[1]);
    // addTimeIntPenalty's sample: step = T_i * (1 / R), s1 = j step, pos = c^T beta0 (a sum from 0 in ascending powers)
    const double step = blob[L.off_T + i] * (1.0 / R);
    const double s1 = j * step, s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2, s5 = s4 * s1;
    const double b0[6] = {1.0, s1, s2, s3, s4, s5};
    const double *c = blob + L.off_c + 18 * i;
    double pos[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        double a = 0.0;
#pragma unroll
        for (int q = 0; q < 6; ++q) a += c[6 * d + q] * b0[q];
        pos[d] = a;
    }
    const double yaw = pos[2];
    double sy, cy;
    dev::sincos_portable(yaw, sy, cy);
    const int size[3] = {A.X, A.Y, A.Z};
    int idx[3][2];
    map_index_box(pos, A.half, A.lo, A.hi, size, A.res, idx);
    const int nx = idx[0][1] - idx[0][0] + 1, ny = idx[1][1] - idx[1][0] + 1, nz = idx[2][1] - idx[2][0] + 1;
    const int64_t cells = (int64_t)nx * ny * nz;
    double costp = 0.0, gpx = 0.0, gpy = 0.0, gyaw = 0.0;
    for (int64_t base = 0; base < cells; base += 32) {
        const int64_t q = base + lane;
        double t[4] = {0.0, 0.0, 0.0, 0.0};
        bool act = false;
        if (q < cells) {
            const int kz = (int)(q % nz);
            const int64_t r = q / nz;
            const int jy = (int)(r % ny) + idx[1][0], ix = (int)(r / ny) + idx[0][0], k = kz + idx[2][0];
            const int fy = jy + A.h;
            const unsigned char byte = A.map[(size_t)k * A.layer + (size_t)(ix + A.h) * A.row_bytes + fy / 8];
            if (byte & (0x80u >> (fy % 8))) {
                // getGridCubeCenter: (index + 0.5) res + boundary_min, never contracted
                const double cx = __dadd_rn(__dmul_rn((double)ix + 0.5, A.res), A.lo[0]);
                const double cyy = __dadd_rn(__dmul_rn((double)jy + 0.5, A.res), A.lo[1]);
                const double cz = __dadd_rn(__dmul_rn((double)k + 0.5, A.res), A.lo[2]);
                // p_minus_x = c - pos (its z: c_z - yaw), p_rel = R^T p_minus_x with R = Rz(yaw) (rotate's unset entries 0)
                const double d0 = cx - pos[0], d1 = cyy - pos[1], d2 = cz - yaw;
                const double rx = cy * d0 + sy * d1, ry = -sy * d0 + cy * d1;
                if (!(fabs(rx) > A.half[0] || fabs(ry) > A.half[1] || fabs(d2) > A.half[2])) {
                    double gx, gy;
                    const double sdf = sdf_with_grad1<SHAPE, XFORM>(S, rx, ry, gx, gy);
                    double sdf_cost = -1.0, L1 = 0.0;
                    host::smoothed_l1(A.safety_hor - sdf, 0.01, sdf_cost, L1);
                    if (sdf_cost > 0) {
                        // grad_cost_p_sw's expressions (point_contribution) at St = I
                        const double rg0 = -(cy * gx + (-sy) * gy), rg1 = -(sy * gx + cy * gy);
                        const double w0 = -sy * d0 + cy * d1, w1 = -cy * d0 + -sy * d1;
                        t[0] = sdf_cost;
                        t[1] = -L1 * rg0;
                        t[2] = -L1 * rg1;
                        t[3] = (-L1 * gx) * w0 + (-L1 * gy) * w1;
                        act = true;
                    }
                }
            }
        }
        // the active cells' terms in the cells' order (ascending lane), summed as the reference's loop sums them
        for (unsigned m = __ballot_sync(kFull, act); m; m &= m - 1) {
            const int src = __ffs(m) - 1;
            costp += __shfl_sync(kFull, t[0], src);
            gpx += __shfl_sync(kFull, t[1], src);
            gpy += __shfl_sync(kFull, t[2], src);
            gyaw += __shfl_sync(kFull, t[3], src);
        }
    }
    if (lane == 0) {
        double *o = A.rec + 4 * (pr.rec_off + item);
        o[0] = costp; o[1] = gpx; o[2] = gpy; o[3] = gyaw;
    }
}

template <int SHAPE, bool XFORM>
cudaError_t launch_shape(const PoseArgs &A, const ShapeParams &S, int max_items, cudaStream_t st) {
    const dim3 grid((unsigned)((max_items + kPoseWarps - 1) / kPoseWarps), (unsigned)A.n);
    k_pose<SHAPE, XFORM><<<grid, kPoseWarps * 32, 0, st>>>(A, S);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_pose(const PoseArgs &A, const ShapeParams &S, int max_items, cudaStream_t st) {
    if (A.n <= 0 || max_items <= 0) return cudaSuccess;
    // the mesh functor is refused by svsdf_set_pose_penalty
    return dispatch_shape<ShapeSet::no_mesh>(S, [&](auto id, auto xf) { return launch_shape<id.value, xf.value>(A, S, max_items, st); });
}

}  // namespace SVSDF_NS
}  // namespace svsdf
