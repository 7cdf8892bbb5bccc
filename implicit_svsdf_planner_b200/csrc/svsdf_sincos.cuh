// svsdf_sincos.cuh — device sin/cos/atan2 used on the SVSDF path.
//
// The reference calls the platform libm here (glibc `sin`/`cos` through Eigen::AngleAxisd, sw_manager.hpp:465-474 and
// back_end_optimizer.hpp:1058-1061; `atan2` in SampleSet2D::initSet :80 and Polygon::isCrossRayOnXDir
// Shape.hpp:1374-1375).  libm is a third-party dependency outside the reference project whose last-bit behaviour is
// unspecified, and that last bit decides which way the reference's sign-descent falls at flat minima (DESIGN.md §Parity).
// This build therefore pins ONE algorithm, made only of IEEE-exact operations (+, -, *, /, fma), on both sides — the
// CPU oracle carries its own copy in oracle/portable_sincos.hpp — so the strict build reproduces the oracle bit for bit:
//   sincos : 3-part Cody–Waite reduction of pi/2 with FMA (quadrant by the 1.5*2^52 rounding trick), then the fdlibm
//            minimax coefficients (k_sin.c S1..S6, k_cos.c C1..C6) in Horner form with FMA.  <= 2 ulp on |x| < 1e6,
//            22 FP64 instructions (the libm-style table/branch code paths are avoided on purpose).
//   atan2  : fdlibm e_atan2.c / s_atan.c (argument reduction to 4 intervals, 11-term polynomial), < 1 ulp.
// |x| >= 1e6 or non-finite arguments fall back to the CUDA library (never reached by yaw angles).
// Coefficients sit in __constant__ memory so FP64 instructions take them as constant-bank operands.
#pragma once
#include <cuda_runtime.h>

namespace svsdf {
namespace dev {

static __constant__ double SC_TAB[20] = {
    /* 0 2/pi   */ 0x1.45f306dc9c883p-1,
    /* 1 pio2_hi*/ 0x1.921fb54442d18p+0, /* 2 pio2_mid */ 0x1.1a62633145c07p-54, /* 3 pio2_lo */ -0x1.f1976b7ed8fbcp-110,
    /* 4 magic  */ 6755399441055744.0,   /* 1.5 * 2^52 */
    /* 5 S1 */ -1.66666666666666324348e-01, /* 6 S2 */ 8.33333333332248946124e-03, /* 7 S3 */ -1.98412698298579493134e-04,
    /* 8 S4 */ 2.75573137070700676789e-06, /* 9 S5 */ -2.50507602534068634195e-08, /* 10 S6 */ 1.58969099521155010221e-10,
    /* 11 C1 */ 4.16666666666666019037e-02, /* 12 C2 */ -1.38888888888741095749e-03, /* 13 C3 */ 2.48015872894767294178e-05,
    /* 14 C4 */ -2.75573143513906633035e-07, /* 15 C5 */ 2.08757232129817482790e-09, /* 16 C6 */ -1.13596475577881948265e-11,
    /* 17 */ -0.5, /* 18 */ 1.0, /* 19 */ 0.0};

__device__ __forceinline__ void sincos_portable(double x, double &s, double &c) {
    if (!(fabs(x) < 1.0e6)) {  // also catches NaN / inf
        ::sincos(x, &s, &c);
        return;
    }
    const double v = fma(x, SC_TAB[0], SC_TAB[4]);  // x * 2/pi + 1.5*2^52: integer part lands in the low mantissa bits
    const int q = __double2loint(v);
    const double fn = v - SC_TAB[4];
    double r = fma(fn, -SC_TAB[1], x);
    r = fma(fn, -SC_TAB[2], r);
    r = fma(fn, -SC_TAB[3], r);
    const double z = r * r;
    double ps = fma(z, SC_TAB[10], SC_TAB[9]);
    ps = fma(z, ps, SC_TAB[8]);
    ps = fma(z, ps, SC_TAB[7]);
    ps = fma(z, ps, SC_TAB[6]);
    ps = fma(z, ps, SC_TAB[5]);
    const double sr = fma(r * z, ps, r);
    double pc = fma(z, SC_TAB[16], SC_TAB[15]);
    pc = fma(z, pc, SC_TAB[14]);
    pc = fma(z, pc, SC_TAB[13]);
    pc = fma(z, pc, SC_TAB[12]);
    pc = fma(z, pc, SC_TAB[11]);
    const double cr = fma(z * z, pc, fma(z, SC_TAB[17], SC_TAB[18]));
    const double ss = (q & 1) ? cr : sr;
    const double cc = (q & 1) ? sr : cr;
    s = (q & 2) ? -ss : ss;
    c = ((q + 1) & 2) ? -cc : cc;
}

// fdlibm s_atan.c
static __constant__ double AT_TAB[20] = {
    /* aT[0..10] */ 3.33333333333329318027e-01, -1.99999999998764832476e-01, 1.42857142725034663711e-01,
    -1.11111104054623557880e-01, 9.09088713343650656196e-02, -7.69187620504482999495e-02, 6.66107313738753120669e-02,
    -5.83357013379057348645e-02, 4.97687799461593236017e-02, -3.65315727442169155270e-02, 1.62858201153657823623e-02,
    /* 11..14 atanhi */ 4.63647609000806093515e-01, 7.85398163397448278999e-01, 9.82793723247329054082e-01,
    1.57079632679489655800e+00,
    /* 15..18 atanlo */ 2.26987774529616870924e-17, 3.06161699786838301793e-17, 1.39033110312309984516e-17,
    6.12323399573676603587e-17, 0.0};

__device__ __forceinline__ double atan_portable(double x) {
    const int hx = __double2hiint(x);
    const int ix = hx & 0x7fffffff;
    int id;
    if (ix >= 0x44100000) {  // |x| >= 2^66 (or inf; NaN handled by the caller)
        const double zz = AT_TAB[14] + AT_TAB[18];
        return (hx > 0) ? zz : -zz;
    }
    if (ix < 0x3fdc0000) {  // |x| < 0.4375
        if (ix < 0x3e200000) return x;  // |x| < 2^-29
        id = -1;
    } else {
        x = fabs(x);
        if (ix < 0x3ff30000) {      // |x| < 1.1875
            if (ix < 0x3fe60000) {  // 7/16 <= |x| < 11/16
                id = 0;
                x = (2.0 * x - 1.0) / (2.0 + x);
            } else {  // 11/16 <= |x| < 19/16
                id = 1;
                x = (x - 1.0) / (x + 1.0);
            }
        } else {
            if (ix < 0x40038000) {  // |x| < 2.4375
                id = 2;
                x = (x - 1.5) / (1.0 + 1.5 * x);
            } else {  // 2.4375 <= |x| < 2^66
                id = 3;
                x = -1.0 / x;
            }
        }
    }
    const double z = x * x;
    const double w = z * z;
    const double s1 = z * (AT_TAB[0] + w * (AT_TAB[2] + w * (AT_TAB[4] + w * (AT_TAB[6] + w * (AT_TAB[8] + w * AT_TAB[10])))));
    const double s2 = w * (AT_TAB[1] + w * (AT_TAB[3] + w * (AT_TAB[5] + w * (AT_TAB[7] + w * AT_TAB[9]))));
    if (id < 0) return x - x * (s1 + s2);
    const double zz = AT_TAB[11 + id] - ((x * (s1 + s2) - AT_TAB[15 + id]) - x);
    return (hx < 0) ? -zz : zz;
}

// fdlibm e_atan2.c (finite arguments; anything else goes to the CUDA library)
__device__ __forceinline__ double atan2_portable(double y, double x) {
    const double pi = 3.1415926535897931160E+00, pi_lo = 1.2246467991473531772E-16, pi_o_2 = 1.5707963267948965580E+00;
    if (!(fabs(x) <= 1.79769313486231570815e+308) || !(fabs(y) <= 1.79769313486231570815e+308)) return ::atan2(y, x);
    const int hx = __double2hiint(x), hy = __double2hiint(y);
    const int ix = hx & 0x7fffffff, iy = hy & 0x7fffffff;
    if (x == 1.0) return atan_portable(y);
    const int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);  // 2*sign(x) + sign(y)
    if (y == 0.0) {
        switch (m) {
            case 0:
            case 1: return y;  // atan(+-0, +anything) = +-0
            case 2: return pi;
            default: return -pi;
        }
    }
    if (x == 0.0) return (hy < 0) ? -pi_o_2 : pi_o_2;
    const int k = (iy - ix) >> 20;
    double z;
    if (k > 60) z = pi_o_2 + 0.5 * pi_lo;            // |y/x| > 2^60
    else if (hx < 0 && k < -60) z = 0.0;             // |y|/x < -2^60
    else z = atan_portable(fabs(y / x));
    switch (m) {
        case 0: return z;
        case 1: return -z;
        case 2: return pi - (z - pi_lo);
        default: return (z - pi_lo) - pi;
    }
}

// ---- single precision (the mesh functor's winding number is a FLOAT computation in the reference) -----------------------
// Explicit round-to-nearest intrinsics: never contracted into FMAs, in either build.
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }

// glibc's atanf / atan2f (fdlibm s_atanf.c / e_atan2f.c; "huge" threshold 2^25) — the same code as
// host/fwn_bvh.hpp: atanf_portable / atan2f_portable, which tests compare with the C library bit for bit.
__device__ __forceinline__ float atanf_portable(float x) {
    const float hi[4] = {4.6364760399e-01f, 7.8539812565e-01f, 9.8279368877e-01f, 1.5707962513e+00f};
    const float lo[4] = {5.0121582440e-09f, 3.7748947079e-08f, 3.4473217170e-08f, 7.5497894159e-08f};
    const int hx = __float_as_int(x), ix = hx & 0x7fffffff;
    int id;
    if (ix >= 0x4c000000) {
        if (ix > 0x7f800000) return fadd(x, x);
        return hx > 0 ? fadd(hi[3], lo[3]) : fsub(-hi[3], lo[3]);
    }
    if (ix < 0x3ee00000) {
        if (ix < 0x31000000) return x;
        id = -1;
    } else {
        x = fabsf(x);
        if (ix < 0x3f980000) {
            if (ix < 0x3f300000) { id = 0; x = fdiv(fsub(fmul(2.0f, x), 1.0f), fadd(2.0f, x)); }
            else { id = 1; x = fdiv(fsub(x, 1.0f), fadd(x, 1.0f)); }
        } else {
            if (ix < 0x401c0000) { id = 2; x = fdiv(fsub(x, 1.5f), fadd(1.0f, fmul(1.5f, x))); }
            else { id = 3; x = fdiv(-1.0f, x); }
        }
    }
    const float z = fmul(x, x), w = fmul(z, z);
    float s1 = 1.6285819933e-02f;
    s1 = fadd(4.9768779427e-02f, fmul(w, s1));
    s1 = fadd(6.6610731184e-02f, fmul(w, s1));
    s1 = fadd(9.0908870101e-02f, fmul(w, s1));
    s1 = fadd(1.4285714924e-01f, fmul(w, s1));
    s1 = fmul(z, fadd(3.3333334327e-01f, fmul(w, s1)));
    float s2 = -3.6531571299e-02f;
    s2 = fadd(-5.8335702866e-02f, fmul(w, s2));
    s2 = fadd(-7.6918758452e-02f, fmul(w, s2));
    s2 = fadd(-1.1111110449e-01f, fmul(w, s2));
    s2 = fmul(w, fadd(-2.0000000298e-01f, fmul(w, s2)));
    if (id < 0) return fsub(x, fmul(x, fadd(s1, s2)));
    const float h = (id == 0) ? hi[0] : (id == 1) ? hi[1] : (id == 2) ? hi[2] : hi[3];
    const float l = (id == 0) ? lo[0] : (id == 1) ? lo[1] : (id == 2) ? lo[2] : lo[3];
    const float r = fsub(h, fsub(fsub(fmul(x, fadd(s1, s2)), l), x));
    return hx < 0 ? -r : r;
}
__device__ __forceinline__ float atan2f_portable(float y, float x) {
    const float pi_o_2 = 1.5707963705e+00f, pi = 3.1415927410e+00f, pi_lo = -8.7422776573e-08f;
    const int hx = __float_as_int(x), ix = hx & 0x7fffffff, hy = __float_as_int(y), iy = hy & 0x7fffffff;
    if (ix >= 0x7f800000 || iy >= 0x7f800000) return ::atan2f(y, x);  // inf / nan: not reached by the solid-angle code
    if (hx == 0x3f800000) return atanf_portable(y);
    const int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);
    if (iy == 0) return (m < 2) ? y : (m == 2 ? pi : -pi);
    if (ix == 0) return hy < 0 ? -pi_o_2 : pi_o_2;
    const int k = (iy - ix) >> 23;
    float z;
    if (k > 60) z = fadd(pi_o_2, fmul(0.5f, pi_lo));
    else if (hx < 0 && k < -60) z = 0.0f;
    else z = atanf_portable(fabsf(fdiv(y, x)));
    switch (m) {
        case 0: return z;
        case 1: return -z;
        case 2: return fsub(pi, fsub(z, pi_lo));
        default: return fsub(fsub(z, pi_lo), pi);
    }
}

}  // namespace dev
}  // namespace svsdf
