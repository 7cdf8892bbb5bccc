// svsdf_kernels_shared.cuh — the single-problem kernels every variant shares, so only the rigid units carry them
// (svsdf_kernels_{fast,strict}.cu): the pose table, the finalize, the shape-functor batch kernels, sincos and the FP64 peak.
#pragma once
#include "svsdf_kernels.cuh"

namespace svsdf {
namespace SVSDF_NS {

// one thread per layer-1 sample, then one per pose-window record
__global__ void k_pose_table(double *blob, PoseRec *w2, PoseRec *w3) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int K1 = (int)blob[1];
    if (e < K1) pose_table_entry(blob, (int)e);
    else if (w2) pose_window_entry(blob, w2, w3, e - K1);
}

__global__ void __launch_bounds__(256) k_finalize(const double *partials, int n_blocks, int N, const int *n_inside,
                                                  const double *gsip_contrib, const int *gsip_piece, double *tot,
                                                  unsigned int *ticket, double *out) {
    finalize_body(partials, n_blocks, N, n_inside ? *n_inside : 0, gsip_contrib, gsip_piece, tot, ticket, out, blockIdx.x, gridDim.x);
}

// ------------------------------------------------------------------------------------------------
// Shape-functor batch kernels (BasicShape::getonlySDF / getonlyGrad1 over arrays of body-frame points)
// ------------------------------------------------------------------------------------------------
template <int SHAPE, bool XFORM>
__global__ void k_shape_sdf(const __grid_constant__ ShapeParams S, const double *rel_xy, int64_t n, double *out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = dev::shape_sdf<SHAPE, XFORM>(S, rel_xy[2 * i], rel_xy[2 * i + 1]);
}
template <int SHAPE, bool XFORM>
__global__ void k_shape_grad(const __grid_constant__ ShapeParams S, const double *rel_xy, int64_t n, double *out3) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double rx = rel_xy[2 * i], ry = rel_xy[2 * i + 1];
    double gx, gy;
    if (SHAPE == SH_POLYGON) {
        dev::PolyHit H = dev::polygon_scan(S, rx, ry);
        double vx = rx - H.cx, vy = ry - H.cy;
        double z = vx * vx + vy * vy;
        if (z > 0.0) { double nn = sqrt(z); vx /= nn; vy /= nn; }
        if (H.rs % 2 != 0) { vx = -vx; vy = -vy; }
        gx = vx; gy = vy;
    } else if (SHAPE == SH_CIRCLE) {
        dev::circle_grad1<XFORM>(S, rx, ry, gx, gy);
    } else {
        const double dx = 0.000001;
        double t0 = rx, t1 = ry;
        t0 -= dx;
        double sdfold = dev::shape_sdf<SHAPE, XFORM>(S, t0, t1);
        t0 += 2 * dx;
        double gradx = dev::shape_sdf<SHAPE, XFORM>(S, t0, t1) - sdfold;
        t0 = rx;
        t1 -= dx;
        sdfold = dev::shape_sdf<SHAPE, XFORM>(S, t0, t1);
        t1 += 2 * dx;
        double grady = dev::shape_sdf<SHAPE, XFORM>(S, t0, t1) - sdfold;
        gx = gradx / (2 * dx);
        gy = grady / (2 * dx);
    }
    out3[3 * i] = gx; out3[3 * i + 1] = gy; out3[3 * i + 2] = 0.0;
}

__global__ void k_sincos(const double *x, int64_t n, double *s, double *c) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double sv, cv;
    dev::sincos_portable(x[i], sv, cv);
    s[i] = sv;
    c[i] = cv;
}

// FP64 FMA peak micro-benchmark (roofline denominator; MEASURED_PEAKS.json has no FP64 figure)
__global__ void __launch_bounds__(256) k_fp64_peak(double *out, int iters) {
    double a0 = threadIdx.x * 1e-3, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
    const double m = 0.999999, c = 1e-6;
    for (int i = 0; i < iters; ++i) {
        a0 = fma(a0, m, c); a1 = fma(a1, m, c); a2 = fma(a2, m, c); a3 = fma(a3, m, c);
        a4 = fma(a4, m, c); a5 = fma(a5, m, c); a6 = fma(a6, m, c); a7 = fma(a7, m, c);
    }
    out[(int64_t)blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
}

cudaError_t launch_pose_table(double *blob, int K1, PoseRec *w2, PoseRec *w3, cudaStream_t stream) {
    const int64_t n = K1 + (w2 ? win2_records(K1) : 0) + (w3 ? win3_records(K1) : 0);
    k_pose_table<<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(blob, w2, w3);
    return cudaGetLastError();
}

cudaError_t launch_finalize(const double *partials, int n_blocks, int N, const int *n_inside,
                            const double *gsip_contrib, const int *gsip_piece, double *tot, unsigned int *ticket,
                            double *out, cudaStream_t stream) {
    const int nacc = 19 * N + 1;
    k_finalize<<<(nacc + 7) / 8, 256, 0, stream>>>(partials, n_blocks, N, n_inside, gsip_contrib, gsip_piece, tot,
                                                   ticket, out);
    return cudaGetLastError();
}

template <int SHAPE, bool XFORM>
static cudaError_t launch_shape_fn(const ShapeParams &S, const double *rel_xy, int64_t n, double *out, int grad,
                                   cudaStream_t stream) {
    int grid = (int)((n + 255) / 256);
    if (grad) k_shape_grad<SHAPE, XFORM><<<grid, 256, 0, stream>>>(S, rel_xy, n, out);
    else k_shape_sdf<SHAPE, XFORM><<<grid, 256, 0, stream>>>(S, rel_xy, n, out);
    return cudaGetLastError();
}

cudaError_t launch_shape_eval(const ShapeParams &S, const double *rel_xy, int64_t n, double *out, int grad,
                              cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    return dispatch_shape<ShapeSet::all>(
        S, [&](auto id, auto xf) { return launch_shape_fn<id.value, xf.value>(S, rel_xy, n, out, grad, stream); });
}

cudaError_t launch_sincos(const double *x, int64_t n, double *s, double *c, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    k_sincos<<<(int)((n + 255) / 256), 256, 0, stream>>>(x, n, s, c);
    return cudaGetLastError();
}

cudaError_t launch_fp64_peak(double *out, int grid, int iters, cudaStream_t stream) {
    k_fp64_peak<<<grid, 256, 0, stream>>>(out, iters);
    return cudaGetLastError();
}

}  // namespace SVSDF_NS
}  // namespace svsdf
