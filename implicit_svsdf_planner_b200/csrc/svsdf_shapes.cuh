// svsdf_shapes.cuh — device-side robot-shape SDF functors (2-D, FP64), one template specialisation per
// registry key of the reference (src/utils/include/utils/Shape.hpp; line of each value function cited).
// Operation order follows the reference so that a -fmad=false build differs from the CPU only through
// libm (sin/cos); every function takes the body-frame point AFTER the shape pre-transform.
#pragma once
#include <cuda_runtime.h>

#include <type_traits>
#include <utility>

#include "svsdf_sincos.cuh"
#include "svsdf_types.h"

namespace svsdf {
namespace dev {

// std::max / std::min exactly as libstdc++ defines them (the reference calls these, not fmax/fmin): 1 compare + select
__device__ __forceinline__ double smaxd(double a, double b) { return (a < b) ? b : a; }
__device__ __forceinline__ double smind(double a, double b) { return (b < a) ? b : a; }
__device__ __forceinline__ double clipd(double v, double lo, double hi) { return smaxd(smind(v, hi), lo); }
__device__ __forceinline__ double len2(double x, double y) { return sqrt(x * x + y * y); }

// a / b for a divisor b known at compile time, given rb = RN(1/b): q = RN(a*rb), r = a - b*q (exact, FMA),
// result RN(q + r*rb).  Markstein's correction step: returns the correctly rounded quotient (bit-identical to the
// IEEE division the reference performs; tests/test_gpu_parity.py::test_strict_shape_functors_are_bitwise checks it)
// in 3 FP64 instructions instead of the ~20-instruction generic division sequence.
__device__ __forceinline__ double div_const(double a, double b, double rb) {
    const double q = a * rb;
    const double r = fma(-b, q, a);
    return fma(r, rb, q);
}

// Literal constants of the shape functors live in __constant__ memory so that FP64 instructions read them as
// constant-bank operands (a double immediate otherwise costs two UMOV per use).  Values are the reference's literals;
// derived entries are folded by the host compiler in IEEE double, one rounding per operation, exactly as the
// reference computes them at run time.
namespace kc {
constexpr double star_k1x = 0.809016994375, star_k1y = -0.587785252292, star_r = 2.8, star_rf = 0.6;
constexpr double star_bax = star_rf * (-star_k1y) - 0.0, star_bay = star_rf * star_k1x - 1.0;
constexpr double star_bb = star_bax * star_bax + star_bay * star_bay;
constexpr double trap_k2x = 3.0 - 1.0, trap_k2y = 2.0 * 2.0;
constexpr double trap_kk = trap_k2x * trap_k2x + trap_k2y * trap_k2y;
constexpr double rhom_bb = 1.0 * 1.0 + 4.5 * 4.5;
}  // namespace kc
__constant__ double KSTAR[8] = {kc::star_k1x, kc::star_k1y, kc::star_r, kc::star_bax, kc::star_bay, kc::star_bb,
                                1.0 / kc::star_bb, 2.0};
__constant__ double KHORSE[4] = {1.5, 1.55, 0.20, 0.0};
__constant__ double KMISC[16] = {
    /*0 pie r*/ 3.0, /*1 arc ra*/ 2.3333, /*2 arc rb*/ 0.5, /*3 tunnel whx*/ 2.5, /*4 tunnel why*/ 1.5,
    /*5 cutdisk r*/ 5.0, /*6 cutdisk h*/ 2.0, /*7 trap kk*/ kc::trap_kk, /*8 1/trap kk*/ 1.0 / kc::trap_kk,
    /*9 rhombus by*/ 4.5, /*10 rhombus bb*/ kc::rhom_bb, /*11 1/bb*/ 1.0 / kc::rhom_bb, /*12*/ 0.25, /*13*/ 0.75,
    /*14*/ 0.5, /*15*/ 2.4};

template <int SHAPE>
struct ShapeFn;

// star — Shape.hpp:584-601 (r = 2.8, rf = 0.6)
template <>
struct ShapeFn<SH_STAR> {
    static __device__ __forceinline__ double sdf(const ShapeParams &, double px, double py) {
        const double k1x = KSTAR[0], k1y = KSTAR[1], r = KSTAR[2];
        const double k2x = -k1x, k2y = k1y;
        px = fabs(px);
        double m = KSTAR[7] * smaxd(k1x * px + k1y * py, 0.0);
        px -= m * k1x;
        py -= m * k1y;
        m = KSTAR[7] * smaxd(k2x * px + k2y * py, 0.0);
        px -= m * k2x;
        py -= m * k2y;
        px = fabs(px);
        py -= r;
        const double bax = KSTAR[3], bay = KSTAR[4];  // rf * (-k1.y, k1.x) - (0, 1)
        double h = clipd(div_const(px * bax + py * bay, KSTAR[5], KSTAR[6]), 0.0, r);
        double dx = px - bax * h, dy = py - bay * h;
        return len2(dx, dy) * copysign(1.0, py * bax - px * bay);
    }
};

// sdHorseshoe — Shape.hpp:870-891; cst = (cos 20.5, sin 20.5) computed on the host (:855)
template <>
struct ShapeFn<SH_HORSESHOE> {
    static __device__ __forceinline__ double sdf(const ShapeParams &S, double px, double py) {
        const double r = KHORSE[0], wx = KHORSE[1], wy = KHORSE[2];
        const double cx = S.cst[0], cy = S.cst[1];
        px = fabs(px);
        double l = len2(px, py);
        double qx = -cx * px + cy * py;
        double qy = cy * px + cx * py;
        double px0 = qx;
        if (px0 <= 0 && qy <= 0) qx = l * copysign(1.0, -cx);
        if (px0 <= 0) qy = l;
        qx = qx - wx;
        qy = fabs(qy - r) - wy;
        double tx = smaxd(qx, 0.0), ty = smaxd(qy, 0.0);
        return len2(tx, ty) + smind(0.0, smaxd(qx, qy));
    }
};

// sdPie / sdPie2 — Shape.hpp:1253-1260 / 1294-1301; cst = (cos 43, sin 43) / (cos 1, sin 1)
__device__ __forceinline__ double sd_pie_c(double px, double py, double cx, double cy) {
    const double r = 3.0;
    px = fabs(px);
    double l = len2(px, py) - r;
    double k = clipd(px * cx + py * cy, 0.0, r);
    double dx = px - cx * k, dy = py - cy * k;
    double m = len2(dx, dy);
    return smaxd(l, m * copysign(1.0, cy * px - cx * py));
}
template <>
struct ShapeFn<SH_PIE> {
    static __device__ __forceinline__ double sdf(const ShapeParams &S, double px, double py) {
        return sd_pie_c(px, py, S.cst[0], S.cst[1]);
    }
};
template <>
struct ShapeFn<SH_PIE2> {
    static __device__ __forceinline__ double sdf(const ShapeParams &S, double px, double py) {
        return sd_pie_c(px, py, S.cst[0], S.cst[1]);
    }
};

// sdArc — Shape.hpp:1334-1343; cst = (sin 20, cos 20), ra = 2.3333, rb = 0.5
template <>
struct ShapeFn<SH_ARC> {
    static __device__ __forceinline__ double sdf(const ShapeParams &S, double px, double py) {
        const double scx = S.cst[0], scy = S.cst[1];
        const double ra = 2.3333, rb = 0.5;
        px = fabs(px);
        bool cond = scy * px > scx * py;
        double ax = px - scx * ra, ay = py - scy * ra;
        double dist1 = len2(ax, ay);
        double dist2 = fabs(len2(px, py) - ra);
        return (cond ? dist1 : dist2) - rb;
    }
};

// sdTunnel — Shape.hpp:642-658; wh = (2.5, 1.5)
template <>
struct ShapeFn<SH_TUNNEL> {
    static __device__ __forceinline__ double sdf(const ShapeParams &, double px, double py) {
        const double whx = 2.5, why = 1.5;
        px = fabs(px);
        py = -py;
        double qx = px - whx, qy = py - why;
        double mq = smaxd(qx, 0.0);
        double d1 = mq * mq + qy * qy;
        qx = (py > 0.0) ? qx : len2(px, py) - whx;
        double mqy = smaxd(qy, 0.0);
        double d2 = qx * qx + mqy * mqy;
        double d = sqrt(smind(d1, d2));
        return (smaxd(qx, qy) < 0.0) ? -d : d;
    }
};

// sdCutDisk — Shape.hpp:698-711; r = 5, h = 2; cst[0] = sqrt(r*r - h*h)
template <>
struct ShapeFn<SH_CUTDISK> {
    static __device__ __forceinline__ double sdf(const ShapeParams &S, double px, double py) {
        const double r = 5.0, h = 2.0;
        const double w = S.cst[0];
        px = fabs(px);
        double s = smaxd((h - r) * px * px + w * w * (h + r - 2.0 * py), h * px - w * py);
        if (s < 0.0) return len2(px, py) - r;
        if (px < w) return h - py;
        return len2(px - w, py - h);
    }
};

// sdTrapezoid — Shape.hpp:754-767; r1 = 1, r2 = 3, he = 2
template <>
struct ShapeFn<SH_TRAPEZOID> {
    static __device__ __forceinline__ double sdf(const ShapeParams &, double px, double py) {
        const double r1 = 1.0, r2 = 3.0, he = 2.0;
        const double k1x = r2, k1y = he;
        const double k2x = r2 - r1, k2y = 2.0 * he;
        px = fabs(px);
        double cax = smaxd(0.0, px - ((py < 0.0) ? r1 : r2));
        double cay = fabs(py) - he;
        double t = clipd(div_const((k1x - px) * k2x + (k1y - py) * k2y, KMISC[7], KMISC[8]), 0.0, 1.0);
        double cbx = px - k1x + k2x * t;
        double cby = py - k1y + k2y * t;
        double s = (cbx < 0.0 && cay < 0.0) ? -1.0 : 1.0;
        return s * sqrt(smind(cax * cax + cay * cay, cbx * cbx + cby * cby));
    }
};

// sdRhombus — Shape.hpp:809-826; b = (1, 4.5)
template <>
struct ShapeFn<SH_RHOMBUS> {
    static __device__ __forceinline__ double sdf(const ShapeParams &, double px, double py) {
        const double bx = 1.0, by = 4.5;
        px = fabs(px);
        py = fabs(py);
        double mx = bx - 2.0 * px, my = by - 2.0 * py;
        double h = clipd(div_const(mx * bx - my * by, KMISC[10], KMISC[11]), -1.0, 1.0);
        double hx = 0.5 * bx, hy = 0.5 * by;
        double dx = px - hx * (1.0 - h), dy = py - hy * (1.0 + h);
        double d = len2(dx, dy);
        double sign = signbit(px * by + py * bx - bx * by) ? -1.0 : 1.0;
        return d * sign;
    }
};

// sdHeart — Shape.hpp:939-952 (input / 4, output * 4); cst[0] = sqrt(2.0) / 4.0
template <>
struct ShapeFn<SH_HEART> {
    static __device__ __forceinline__ double sdf(const ShapeParams &S, double px, double py) {
        px = px / 4.0;
        py = py / 4.0;
        px = fabs(px);
        if (py + px > 1.0) return 4 * (len2(px - 0.25, py - 0.75) - S.cst[0]);
        double ax = px - 0.0, ay = py - 1.0;
        double v1 = ax * ax + ay * ay;
        double t = smaxd(px + py, 0.0);
        double bx = px - 0.5 * t, by = py - 0.5 * t;
        double v2 = bx * bx + by * by;
        return 4 * (sqrt(smind(v1, v2)) * copysign(1.0, px - py));
    }
};

// sdRoundedX / bigX — Shape.hpp:988-994 (w = 3, r = 0.25) / 1024-1030 (w = 5, r = 0.25)
__device__ __forceinline__ double sd_roundedx_w(double px, double py, double w, double r) {
    double ax = fabs(px), ay = fabs(py);
    double m = (ax + ay > w) ? (w * 0.5) : (ax + ay) * 0.5;
    return len2(ax - m, ay - m) - r;
}
template <>
struct ShapeFn<SH_ROUNDEDX> {
    static __device__ __forceinline__ double sdf(const ShapeParams &, double px, double py) {
        return sd_roundedx_w(px, py, 3.0, 0.25);
    }
};
template <>
struct ShapeFn<SH_BIGX> {
    static __device__ __forceinline__ double sdf(const ShapeParams &, double px, double py) {
        return sd_roundedx_w(px, py, 5.0, 0.25);
    }
};

// sdRoundedCross — Shape.hpp:1062-1075; h = 1, input / 2, output * 2
template <>
struct ShapeFn<SH_ROUNDEDCROSS> {
    static __device__ __forceinline__ double sdf(const ShapeParams &, double px, double py) {
        const double h = 1.0;
        px = px / 2.0;
        py = py / 2.0;
        const double k = 0.5 * (h + 1.0 / h);
        double ax = fabs(px), ay = fabs(py);
        if (ax < 1.0 && ay < ax * (k - h) + h) return 2 * (k - len2(ax - 1.0, ay - k));
        double d1x = ax - 0.0, d1y = ay - h;
        double d2x = ax - 1.0, d2y = ay - 0.0;
        return 2 * sqrt(smind(d1x * d1x + d1y * d1y, d2x * d2x + d2y * d2y));
    }
};

// sdOrientedVesica — Shape.hpp:1115-1146; a = (2,4), b = (-2,-4), w = 0.8
// cst = (r, d, vx, vy) with r = 0.5*|b-a|, d = 0.5*(r*r - w*w)/w, v = (b-a)/r  (host-computed, same formulas)
template <>
struct ShapeFn<SH_VESICA> {
    static __device__ __forceinline__ double sdf(const ShapeParams &S, double px, double py) {
        const double w = 0.8;
        const double r = S.cst[0], d = S.cst[1], vx = S.cst[2], vy = S.cst[3];
        const double cx = 0.5 * (-2.0 + 2.0), cy = 0.5 * (-4.0 + 4.0);
        px = px / 1.0;
        py = py / 1.0;
        double ux = px - cx, uy = py - cy;
        double qx = 0.5 * fabs(vy * ux + vx * uy);
        double qy = 0.5 * fabs(-vx * ux + vy * uy);
        double hx, hy, hz;
        if (r * qx < d * (qy - r)) {
            hx = 0.0; hy = r; hz = 0.0;
        } else {
            hx = -d; hy = 0.0; hz = d + w;
        }
        return 1.0 * (len2(qx - hx, qy - hy) - hz);
    }
};

// sdMoon — Shape.hpp:1202-1214; d = 0.8, ra = 3, rb = 2.4; cst = (a, b) host-computed
template <>
struct ShapeFn<SH_MOON> {
    static __device__ __forceinline__ double sdf(const ShapeParams &S, double qx, double qy) {
        const double d = 0.8, ra = 3.0, rb = 2.4;
        const double a = S.cst[0], b = S.cst[1];
        qy = fabs(qy);
        bool cond = d * (qx * b - qy * a) > d * d * smaxd(b - qy, 0.0);
        double dist1 = len2(qx - a, qy - b);
        double dist2 = smaxd(len2(qx, qy) - ra, -len2(qx - d, qy - 0.0) + rb);
        return cond ? dist1 : dist2;
    }
};

// sdUnevenCapsule — Shape.hpp:531-543; r1 = 2, r2 = 1, h = 5; cst = (b, a) host-computed
template <>
struct ShapeFn<SH_UNEVENCAPSULE> {
    static __device__ __forceinline__ double sdf(const ShapeParams &S, double px, double py) {
        const double r1 = 2.0, r2 = 1.0, h = 5.0;
        const double b = S.cst[0], a = S.cst[1];
        px = fabs(px);
        double k = px * (-b) + py * a;
        if (k < 0.0) return len2(px, py) - r1;
        if (k > a * h) return len2(px - 0.0, py - h) - r2;
        return px * a + py * b - r1;
    }
};

// Circle — Shape.hpp:476-480
template <>
struct ShapeFn<SH_CIRCLE> {
    static __device__ __forceinline__ double sdf(const ShapeParams &S, double px, double py) {
        return len2(px, py) - S.radius;
    }
};

// Polygon fallback — Shape.hpp:1370-1400 (edge helpers), 1448-1476 (SDF), 1508-1534 (analytic gradient).
// Ignores trans/Rotate, like the reference (:1451).
struct PolyHit {
    double dis, cx, cy;
    int rs;
};
__device__ __forceinline__ PolyHit polygon_scan(const ShapeParams &S, double qx, double qy) {
    const double PI = 3.14159265358979323846;
    PolyHit H{1e9, 0.0, 0.0, 0};
#pragma unroll 1
    for (int i = 0; i < S.poly_n; ++i) {
        double sx = S.poly_sx[i], sy = S.poly_sy[i], ex = S.poly_ex[i], ey = S.poly_ey[i];
        double vx = ex - sx, vy = ey - sy;
        double wx = qx - sx, wy = qy - sy;
        double t = (wx * vx + wy * vy) / (vx * vx + vy * vy);
        if (t < 0.0) t = 0.0;
        else if (t > 1.0) t = 1.0;
        double cx = sx + t * vx, cy = sy + t * vy;
        double dis = len2(qx - cx, qy - cy);
        if (dis < H.dis) {
            H.dis = dis; H.cx = cx; H.cy = cy;
        }
        // Crossing test (Shape.hpp:1461-1470): with both polar angles mapped to [0, 2 pi), |ths - the| >= pi.  In exact terms:
        // a = s - q and b = e - q lie on different sides of the horizontal through q, and b is at least a half turn ahead of a
        // (sin of the turn = cross(a, b) / |a||b| <= 0 when a is above, >= 0 when a is below); equal sides never reach pi.  The two
        // atan2 calls are needed only where their rounding (a few 1e-16 rad) could decide: an offset exactly on the horizontal, or
        // a and b within 1e-9 rad of (anti)parallel.  Everywhere else the sign tests give the same answer as the angles.
        const double ax = sx - qx, ay = sy - qy, bx = ex - qx, by = ey - qy;
        const double cr = ax * by - ay * bx;
        bool crossing;
        if (ay != 0.0 && by != 0.0 && fabs(cr) > 1e-9 * ((fabs(ax) + fabs(ay)) * (fabs(bx) + fabs(by)))) {
            crossing = ((ay > 0.0) != (by > 0.0)) && ((ay > 0.0) ? (cr < 0.0) : (cr > 0.0));
        } else {
            double ths = atan2_portable(ay, ax), the = atan2_portable(by, bx);
            ths = (ths < 0.0) ? (ths + 2 * PI) : ths;
            the = (the < 0.0) ? (the + 2 * PI) : the;
            const double d1 = fabs(ths - the);
            crossing = !(d1 < PI);
        }
        if (crossing) H.rs++;
    }
    return H;
}
template <>
struct ShapeFn<SH_POLYGON> {
    static __device__ __forceinline__ double sdf(const ShapeParams &S, double qx, double qy) {
        PolyHit H = polygon_scan(S, qx, qy);
        return (H.rs % 2 == 0) ? H.dis : -H.dis;
    }
};

// Triangle-mesh functor — BasicShape::getonlySDF_igl (Shape.hpp:332-340): sdf = (1 - 2 w) * sqrt(d2).
//   w  = igl::fast_winding_number(fwn_bvh, 2.0, p) (fast_winding_number.cpp:439-457): the HDK's UT_SolidAngle<float,float>,
//        a 4-way hierarchy with order-2 expansions, evaluated in SINGLE precision.  The hierarchy is built on the host
//        (host/fwn_bvh.hpp, bitwise the reference's tree and coefficients); fwn_solid_angle() below walks it exactly as
//        computeSolidAngle's recursive traverseVector does (FastWindingNumberForSoups.h:7149-7284): per node the four child
//        expansions summed left to right, then the descended children's results summed left to right in slot order — an
//        explicit stack of frames stands in for the recursion.  Every float operation is a *_rn intrinsic (no FMA), atan2f
//        is the pinned fdlibm code: w equals the reference's value BIT FOR BIT (tests/test_gpu_mesh.py).
//   d2 = squared distance to the closest triangle: igl::AABB::squared_distance (AABB.cpp:1130-1200) is a pruned minimum over
//        point_simplex_squared_distance (point_simplex_squared_distance.cpp:43-116, Ericson's closest point), in double.
//        closest_sqr_distance() prunes over the SAME 4-way tree's child boxes (rounded outwards, so they contain the double
//        vertices): a subtree is skipped only when its box is provably farther than the best face so far, hence the result
//        is the plain minimum over all faces — the same number the reference's own pruned search returns.
// The query is (qx, qy, 0): the path zeroes the z of both the pose and the point (sw_manager.hpp:767,
// back_end_optimizer.hpp:791).
template <>
struct ShapeFn<SH_MESH> {
    // UTsignedSolidAngleTri (FastWindingNumberForSoups.h:6071-6110), float
    static __device__ __forceinline__ float tri_solid_angle(const float4 *T, float qx, float qy, float qz) {
        const float4 t0 = __ldg(T), t1 = __ldg(T + 1), t2 = __ldg(T + 2);  // a.xyz b.x | b.yz c.xy | c.z - - -
        float a0 = fsub(t0.x, qx), a1 = fsub(t0.y, qy), a2 = fsub(t0.z, qz);
        float b0 = fsub(t0.w, qx), b1 = fsub(t1.x, qy), b2 = fsub(t1.y, qz);
        float c0 = fsub(t1.z, qx), c1 = fsub(t1.w, qy), c2 = fsub(t2.x, qz);
        const float al = __fsqrt_rn(fadd(fadd(fmul(a0, a0), fmul(a1, a1)), fmul(a2, a2)));
        const float bl = __fsqrt_rn(fadd(fadd(fmul(b0, b0), fmul(b1, b1)), fmul(b2, b2)));
        const float cl = __fsqrt_rn(fadd(fadd(fmul(c0, c0), fmul(c1, c1)), fmul(c2, c2)));
        if (al == 0.0f || bl == 0.0f || cl == 0.0f) return 0.0f;
        const float ia = fdiv(1.0f, al), ib = fdiv(1.0f, bl), ic = fdiv(1.0f, cl);
        a0 = fmul(a0, ia); a1 = fmul(a1, ia); a2 = fmul(a2, ia);
        b0 = fmul(b0, ib); b1 = fmul(b1, ib); b2 = fmul(b2, ib);
        c0 = fmul(c0, ic); c1 = fmul(c1, ic); c2 = fmul(c2, ic);
        const float u0 = fsub(b0, a0), u1 = fsub(b1, a1), u2 = fsub(b2, a2);
        const float v0 = fsub(c0, a0), v1 = fsub(c1, a1), v2 = fsub(c2, a2);
        const float n0 = fsub(fmul(u1, v2), fmul(u2, v1)), n1 = fsub(fmul(u2, v0), fmul(u0, v2)), n2 = fsub(fmul(u0, v1), fmul(u1, v0));
        const float num = fadd(fadd(fmul(a0, n0), fmul(a1, n1)), fmul(a2, n2));
        if (num == 0.0f) return 0.0f;
        const float dab = fadd(fadd(fmul(a0, b0), fmul(a1, b1)), fmul(a2, b2));
        const float dac = fadd(fadd(fmul(a0, c0), fmul(a1, c1)), fmul(a2, c2));
        const float dbc = fadd(fadd(fmul(b0, c0), fmul(b1, c1)), fmul(b2, c2));
        const float den = fadd(fadd(fadd(1.0f, dab), dac), dbc);
        return fmul(2.0f, atan2f_portable(num, den));
    }
    // one node: the four children's order-2 expansions (computeSolidAngle's per-lane arithmetic, :7190-7255), summed left to
    // right; bit i of `descend` = child i has to be entered.  Row r, lane i of the node record is D[4 * r + i].  The loop
    // is NOT unrolled and this function has ONE call site: the traversal's code has to stay resident in the instruction cache
    // while the lanes of a warp sit in different parts of it.
    static __device__ __forceinline__ void node_terms(const float *D, float qx, float qy, float qz, float acc2, float &sum, unsigned &descend) {
        descend = 0;
        sum = 0.0f;
#pragma unroll 1
        for (int i = 0; i < 4; ++i) {
            const float *r = D + i;
#define R_(k) __ldg(r + 4 * (k))
            float q0 = fsub(qx, R_(1)), q1 = fsub(qy, R_(2)), q2 = fsub(qz, R_(3));
            const float ql2 = fadd(fadd(fmul(q0, q0), fmul(q1, q1)), fmul(q2, q2));
            float om = 0.0f;
            // a child inside its own accuracy radius is entered whatever its expansion says (the reference evaluates all four
            // lanes in SIMD and discards this one): skip the ~150 operations
            bool use = !(ql2 <= fmul(R_(0), acc2));
            if (use) {
                const float m2 = fdiv(1.0f, ql2), m1 = __fsqrt_rn(m2);
                q0 = fmul(q0, m1); q1 = fmul(q1, m1); q2 = fmul(q2, m1);
                om = fmul(-m2, fadd(fadd(fmul(q0, R_(4)), fmul(q1, R_(5))), fmul(q2, R_(6))));
                const float s0 = fmul(q0, q0), s1 = fmul(q1, q1), s2 = fmul(q2, q2);
                const float m3 = fmul(m2, m1);
                const float r7 = R_(7), r8 = R_(8), r9 = R_(9);
                const float in1 = fadd(fadd(fadd(fadd(fadd(fmul(s0, r7), fmul(s1, r8)), fmul(s2, r9)), fmul(fmul(q0, q1), R_(10))),
                                            fmul(fmul(q0, q2), R_(12))), fmul(fmul(q1, q2), R_(11)));
                const float o1 = fmul(m3, fsub(fadd(fadd(r7, r8), r9), fmul(3.0f, in1)));
                om = fadd(om, o1);
                const float c0 = fmul(s0, q0), c1 = fmul(s1, q1), c2 = fmul(s2, q2);
                const float m4 = fmul(m2, m2);
                const float r13 = R_(13), r14 = R_(14), r15 = R_(15), r17 = R_(17), r18 = R_(18), r19 = R_(19), r20 = R_(20), r21 = R_(21),
                            r22 = R_(22);
                const float t00 = fadd(r20, r21), t01 = fadd(r22, r17), t02 = fadd(r18, r19);
                const float t10 = fadd(fmul(q1, r17), fmul(q2, r18)), t11 = fadd(fmul(q2, r19), fmul(q0, r20)),
                            t12 = fadd(fmul(q0, r21), fmul(q1, r22));
                const float da = fadd(fadd(fmul(q0, fadd(fmul(3.0f, r13), t00)), fmul(q1, fadd(fmul(3.0f, r14), t01))),
                                      fmul(q2, fadd(fmul(3.0f, r15), t02)));
                const float db = fadd(fadd(fadd(fadd(fmul(c0, r13), fmul(c1, r14)), fmul(c2, r15)), fmul(fmul(fmul(q0, q1), q2), R_(16))),
                                      fadd(fadd(fmul(s0, t10), fmul(s1, t11)), fmul(s2, t12)));
                const float o2 = fmul(m4, fsub(fmul(1.5f, da), fmul(7.5f, db)));
                om = fadd(om, o2);
                use = isfinite(om);
            }
#undef R_
            const float a = use ? om : 0.0f;
            sum = (i == 0) ? a : fadd(sum, a);  // ((a0 + a1) + a2) + a3; all four entered -> 0, as the reference's early return
            if (!use) descend |= 1u << i;
        }
    }
    static __device__ __noinline__ float fwn_solid_angle(const ShapeParams &S, float qx, float qy, float qz) {
        const float acc2 = 4.0f;  // accuracy_scale 2.0 (Shape.hpp:337), squared
        const float4 *trif = reinterpret_cast<const float4 *>(S.fwn_trif);
        // frame d: node, expansion sum, descend mask (bits 0-3) | next slot (bits 4-6), partial sum of the slots done so far
        int f_node[kFwnMaxDepth];
        float f_sum[kFwnMaxDepth], f_ps[kFwnMaxDepth];
        unsigned f_st[kFwnMaxDepth];
        int d = -1, next = 0;
        float ret = 0.0f;
        bool have_ret = false;
        // A valid hierarchy ends within 2 nn - 1 iterations (every node entered once, returned from once); past the bound the
        // hierarchy is corrupt and the result is NaN rather than a spinning warp.  The bounded loop is also what the sm_90a
        // code of the standalone shape kernel needs: built without this exit, k_shape_sdf<SH_MESH> never returned on the H100.
        const int max_iter = 4 * (S.fwn_nn + 1);
#pragma unroll 1
        for (int iter = 0;; ++iter) {
            if (iter > max_iter) return __int_as_float(0x7fc00000);
            if (!have_ret) {  // enter node `next` as a new frame
                ++d;
                f_node[d] = next;
                f_ps[d] = 0.0f;
                node_terms(S.fwn_data + 92 * (size_t)next, qx, qy, qz, acc2, f_sum[d], f_st[d]);
            }
            const unsigned st = f_st[d];
            int s = (int)(st >> 4);
            float ps = f_ps[d];
            if (have_ret) {  // a child frame has just returned into slot s
                ps = (s == 0) ? ret : fadd(ps, ret);
                ++s;
                have_ret = false;
            }
            bool pushed = false;
#pragma unroll 1
            while (s < 4) {
                float v = 0.0f;
                if ((st >> s) & 1u) {
                    const unsigned c = __ldg(S.fwn_child + 4 * (size_t)f_node[d] + s);
                    if (c & 0x80000000u) {
                        if (c == 0xffffffffu) break;  // no more children: the remaining slots are not summed
                        if (d + 1 < kFwnMaxDepth) {
                            f_st[d] = (st & 0xfu) | ((unsigned)s << 4);
                            f_ps[d] = ps;
                            next = (int)(c & 0x7fffffffu);
                            pushed = true;
                            break;
                        }
                    } else {
                        v = tri_solid_angle(trif + 3 * (size_t)c, qx, qy, qz);
                    }
                }
                ps = (s == 0) ? v : fadd(ps, v);
                ++s;
            }
            if (pushed) continue;
            ret = fadd(f_sum[d], ps);
            if (d == 0) return ret;
            --d;
            have_ret = true;
        }
    }
    // Single-precision LOWER bound of the squared distance from (qx, qy, 0) to a child box.  Record (6 floats, built on the
    // host): lo x, lo y, hi x, hi y (rounded outwards so the box contains the double vertices), dz2 = the squared z gap of the
    // box to the plane z = 0 rounded down, pad.  qf = float(q) is off by <= 2^-24 |q| and lo - qf rounds by <= 2^-24 (|lo| + |qf|):
    // subtracting e = 2.4e-7 (|qf| + M) (M >= every |box coordinate|; twice the worst case) makes each gap a lower bound, and the
    // factor (1 - 4e-7) covers the five roundings of the sum of squares.
    static __device__ __forceinline__ float box_lb2(const float *b, float qxf, float qyf, float ex, float ey) {
        const float2 lo = __ldg(reinterpret_cast<const float2 *>(b)), hi = __ldg(reinterpret_cast<const float2 *>(b) + 1);
        const float dz2 = __ldg(b + 4);
        const float dx = fmaxf(fmaxf(lo.x - qxf, qxf - hi.x) - ex, 0.0f);
        const float dy = fmaxf(fmaxf(lo.y - qyf, qyf - hi.y) - ey, 0.0f);
        return (dx * dx + dy * dy + dz2) * 0.9999996f;
    }
    // Squared distance from p to triangle (a, b, c): ClosestBaryPtPointTriangle (point_simplex_squared_distance.cpp:43-106).
    // The reference walks the seven Voronoi regions with early returns; here the region is decided first (same conditions,
    // same order: A, B, AB, C, AC, BC, interior) and the ONE division the chosen region needs is done once — lane for lane
    // the same IEEE operations as the early-return form (the oracle's), but a warp whose lanes fall into different regions
    // no longer executes four divergent division sequences.
    static __device__ __forceinline__ double sqr_distance(double ax, double ay, double az, double bx, double by, double bz,
                                                          double cx, double cy, double cz, double px, double py, double pz) {
        const double abx = bx - ax, aby = by - ay, abz = bz - az;
        const double acx = cx - ax, acy = cy - ay, acz = cz - az;
        const double apx = px - ax, apy = py - ay, apz = pz - az;
        const double d1 = (abx * apx + aby * apy) + abz * apz;
        const double d2 = (acx * apx + acy * apy) + acz * apz;
        const double bpx = px - bx, bpy = py - by, bpz = pz - bz;
        const double d3 = (abx * bpx + aby * bpy) + abz * bpz;
        const double d4 = (acx * bpx + acy * bpy) + acz * bpz;
        const double cpx = px - cx, cpy = py - cy, cpz = pz - cz;
        const double d5 = (abx * cpx + aby * cpy) + abz * cpz;
        const double d6 = (acx * cpx + acy * cpy) + acz * cpz;
        const double vc = d1 * d4 - d3 * d2, vb = d5 * d2 - d1 * d6, va = d3 * d6 - d5 * d4;
        const double e43 = d4 - d3, e56 = d5 - d6;
        const bool a_ne_b = (ax != bx) || (ay != by) || (az != bz);
        const bool rA = d1 <= 0.0 && d2 <= 0.0;
        const bool rB = !rA && d3 >= 0.0 && d4 <= d3;
        const bool rAB = !rA && !rB && a_ne_b && vc <= 0.0 && d1 >= 0.0 && d3 <= 0.0;
        const bool done3 = rA || rB || rAB;
        const bool rC = !done3 && d6 >= 0.0 && d5 <= d6;
        const bool rAC = !done3 && !rC && vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0;
        const bool done5 = done3 || rC || rAC;
        const bool rBC = !done5 && va <= 0.0 && e43 >= 0.0 && e56 >= 0.0;
        const bool rIN = !done5 && !rBC;
        const double num = rAB ? d1 : rAC ? d2 : rBC ? e43 : 1.0;
        const double den = rAB ? (d1 - d3) : rAC ? (d2 - d6) : rBC ? (e43 + e56) : rIN ? ((va + vb) + vc) : 1.0;
        const double r = num / den;
        // edge regions: base + r * dir; interior: (a + ab * v) + ac * w with v = vb * r, w = vc * r
        const double bsx = rBC ? bx : ax, bsy = rBC ? by : ay, bsz = rBC ? bz : az;
        const double drx = rAB ? abx : rAC ? acx : (cx - bx), dry = rAB ? aby : rAC ? acy : (cy - by), drz = rAB ? abz : rAC ? acz : (cz - bz);
        const double v = vb * r, w = vc * r;
        const double c1 = rIN ? v : r;
        const double ux = rIN ? abx : drx, uy = rIN ? aby : dry, uz = rIN ? abz : drz;
        double qx = bsx + c1 * ux, qy = bsy + c1 * uy, qz = bsz + c1 * uz;  // a + v * ab  ==  ax + abx * v
        if (rIN) { qx = qx + acx * w; qy = qy + acy * w; qz = qz + acz * w; }
        if (rA) { qx = ax; qy = ay; qz = az; }
        if (rB) { qx = bx; qy = by; qz = bz; }
        if (rC) { qx = cx; qy = cy; qz = cz; }
        const double ex = px - qx, ey = py - qy, ez = pz - qz;
        return (ex * ex + ey * ey) + ez * ez;
    }
    // Nearest-first descent over the hierarchy's child boxes.  Per node: the four children's float lower bounds; faces whose
    // bound does not exceed the best squared distance so far are evaluated (exact, double); of the internal children that
    // survive, the nearest is entered directly and the others go on an explicit stack of (node, bound).  A subtree or a face is
    // skipped only if its LOWER bound exceeds best * (1 + 1e-12) rounded up to float: conservative, so the minimum over the
    // visited faces is the minimum over ALL faces, bit for bit (the oracle takes the plain minimum).  Children are picked from
    // registers with selects (no dynamically indexed local arrays), and sqr_distance has one call site.
    static __device__ __forceinline__ float sel4(int s, float a, float b, float c, float d) { return s == 0 ? a : s == 1 ? b : s == 2 ? c : d; }
    static __device__ __forceinline__ unsigned sel4(int s, unsigned a, unsigned b, unsigned c, unsigned d) { return s == 0 ? a : s == 1 ? b : s == 2 ? c : d; }
    static __device__ __noinline__ double closest_sqr_distance(const ShapeParams &S, double qx, double qy) {
        constexpr int kStack = 3 * kFwnMaxDepth + 4;
        int st_node[kStack];
        float st_lb[kStack];
        int top = 0;
        const float INF = __int_as_float(0x7f800000);
        const float qxf = (float)qx, qyf = (float)qy;
        const float ex = 2.4e-7f * (fabsf(qxf) + S.fwn_boxmag), ey = 2.4e-7f * (fabsf(qyf) + S.fwn_boxmag);
        double best = __longlong_as_double(0x7ff0000000000000LL);
        float bestf = INF;  // >= best * (1 + 1e-12)
        int node = 0;
        // every node is processed at most once and every stack entry popped at most once: <= 2 nn + 1 iterations on a valid
        // hierarchy (bounded for the same two reasons as fwn_solid_angle's loop)
        const int max_iter = 4 * (S.fwn_nn + 1);
#pragma unroll 1
        for (int iter = 0;; ++iter) {
            if (iter > max_iter) return __longlong_as_double(0x7ff8000000000000LL);
            if (node < 0) {
                if (top == 0) break;
                --top;
                node = st_node[top];
                if (st_lb[top] > bestf) { node = -1; continue; }
            }
            const uint4 cw = __ldg(reinterpret_cast<const uint4 *>(S.fwn_child) + node);
            const float *cb = S.fwn_cbox + 24 * (size_t)node;
            const float l0 = box_lb2(cb, qxf, qyf, ex, ey);
            const float l1 = (cw.y == 0xffffffffu) ? INF : box_lb2(cb + 6, qxf, qyf, ex, ey);
            const float l2 = (cw.z == 0xffffffffu) ? INF : box_lb2(cb + 12, qxf, qyf, ex, ey);
            const float l3 = (cw.w == 0xffffffffu) ? INF : box_lb2(cb + 18, qxf, qyf, ex, ey);
            // faces first (they tighten the bound before anything is entered)
#pragma unroll 1
            for (int s = 0; s < 4; ++s) {
                const unsigned c = sel4(s, cw.x, cw.y, cw.z, cw.w);
                if ((c & 0x80000000u) || sel4(s, l0, l1, l2, l3) > bestf) continue;
                const double *t = S.mesh_tri + (size_t)c * kMeshStride;
                const double2 v0 = __ldg(reinterpret_cast<const double2 *>(t)), v1 = __ldg(reinterpret_cast<const double2 *>(t) + 1),
                              v2 = __ldg(reinterpret_cast<const double2 *>(t) + 2), v3 = __ldg(reinterpret_cast<const double2 *>(t) + 3);
                const double cz = __ldg(t + 8);
                const double dd = sqr_distance(v0.x, v0.y, v1.x, v1.y, v2.x, v2.y, v3.x, v3.y, cz, qx, qy, 0.0);
                if (dd < best) { best = dd; bestf = __double2float_ru(dd * (1.0 + 1e-12)); }
            }
            // internal children still in range: nearest next, the rest stacked
            const bool i0 = (cw.x & 0x80000000u) && l0 <= bestf, i1 = (cw.y & 0x80000000u) && cw.y != 0xffffffffu && l1 <= bestf,
                       i2 = (cw.z & 0x80000000u) && cw.z != 0xffffffffu && l2 <= bestf, i3 = (cw.w & 0x80000000u) && cw.w != 0xffffffffu && l3 <= bestf;
            const float m0 = i0 ? l0 : INF, m1 = i1 ? l1 : INF, m2 = i2 ? l2 : INF, m3 = i3 ? l3 : INF;
            int near = -1;
            float ml = INF;
            if (i0) { near = 0; ml = m0; }
            if (i1 && m1 < ml) { near = 1; ml = m1; }
            if (i2 && m2 < ml) { near = 2; ml = m2; }
            if (i3 && m3 < ml) { near = 3; ml = m3; }
            if (i0 && near != 0 && top < kStack) { st_node[top] = (int)(cw.x & 0x7fffffffu); st_lb[top] = l0; ++top; }
            if (i1 && near != 1 && top < kStack) { st_node[top] = (int)(cw.y & 0x7fffffffu); st_lb[top] = l1; ++top; }
            if (i2 && near != 2 && top < kStack) { st_node[top] = (int)(cw.z & 0x7fffffffu); st_lb[top] = l2; ++top; }
            if (i3 && near != 3 && top < kStack) { st_node[top] = (int)(cw.w & 0x7fffffffu); st_lb[top] = l3; ++top; }
            node = (near < 0) ? -1 : (int)(sel4(near, cw.x, cw.y, cw.z, cw.w) & 0x7fffffffu);
        }
        return best;
    }
    static __device__ __forceinline__ double sdf(const ShapeParams &S, double qx, double qy) {
        const double PI = 3.1415926535897932384626433832795;  // igl::PI
        const float omega = fwn_solid_angle(S, (float)qx, (float)qy, 0.0f);
        const double w = (double)omega / (4.0 * PI);
        const double best = closest_sqr_distance(S, qx, qy);
        const double s = 1. - 2. * w;
        return s * sqrt(best);
    }
};

// ((pos_rel - trans) * Rotate).head(2): row-vector times matrix (Shape.hpp:281-294 and e.g. :586).
// With has_xform == 0 (trans = 0, Rotate = I) the product is the identity bit-for-bit and is skipped.
template <int SHAPE, bool XFORM>
__device__ __forceinline__ double shape_sdf(const ShapeParams &S, double rx, double ry) {
    if (SHAPE != SH_POLYGON && SHAPE != SH_MESH && XFORM) {
        double v0 = rx - S.trans[0], v1 = ry - S.trans[1];
        rx = v0 * S.rot[0] + v1 * S.rot[2];
        ry = v0 * S.rot[1] + v1 * S.rot[3];
    }
    return ShapeFn<SHAPE>::sdf(S, rx, ry);
}

// Circle overrides getonlyGrad1 (Shape.hpp:487-497): the normalised ((p - trans) * Rotate).head(2), no finite difference
template <bool XFORM>
__device__ __forceinline__ void circle_grad1(const ShapeParams &S, double rx, double ry, double &gx, double &gy) {
    if (XFORM) {
        double v0 = rx - S.trans[0], v1 = ry - S.trans[1];
        rx = v0 * S.rot[0] + v1 * S.rot[2];
        ry = v0 * S.rot[1] + v1 * S.rot[3];
    }
    double z = rx * rx + ry * ry;
    if (z > 0.0) {  // Eigen normalize(): divides by sqrt(squaredNorm)
        double n = sqrt(z);
        rx /= n; ry /= n;
    }
    gx = rx; gy = ry;
}

}  // namespace dev

// The functors a kernel family is compiled for.  Each set's value is one past its last id (the ids are contiguous): every functor, every
// functor but the mesh (the pose penalty), or the analytic ones (the A* front end: the reference has no rotated kernels for the others).
enum class ShapeSet { all = SH_COUNT, no_mesh = SH_MESH, analytic = SH_POLYGON };

template <int ID, class F>
cudaError_t call_shape(const ShapeParams &S, F &f) {
    if constexpr (ID < SH_POLYGON)  // only the analytic functors apply the pre-transform
        if (S.has_xform) return f(std::integral_constant<int, ID>{}, std::true_type{});
    return f(std::integral_constant<int, ID>{}, std::false_type{});
}
template <class F, int... IDS>
cudaError_t dispatch_ids(const ShapeParams &S, F &f, std::integer_sequence<int, IDS...>) {
    cudaError_t e = cudaErrorInvalidValue;
    (void)((S.id == IDS && ((e = call_shape<IDS>(S, f)), true)) || ...);
    return e;
}

// Host-side shape dispatch of every launcher: f(id, xform) with S's functor id and pre-transform flag as std::integral_constant, so
// that f can instantiate its kernel on them.  An id outside SET returns cudaErrorInvalidValue.
template <ShapeSet SET, class F>
cudaError_t dispatch_shape(const ShapeParams &S, F &&f) {
    return dispatch_ids(S, f, std::make_integer_sequence<int, (int)SET>{});
}

}  // namespace svsdf
