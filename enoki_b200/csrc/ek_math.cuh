/*
 * ek_math.cuh -- device math with the numerics of the reference's CPU path.
 *
 * The reference's own GPU backend maps exp/log/sin/cos/rcp/rsqrt to PTX
 * `.approx.ftz` instructions (include/enoki/cuda.h:433-467).  BASELINE.json's
 * north star asks for parity with the reference's *CPU* path instead, so these
 * are the Cephes-derived polynomials of include/enoki/array_math.h evaluated with
 * the same Estrin groupings (array_math.h:25-105) and explicit IEEE add/mul/fma
 * intrinsics (never contracted, no flush-to-zero), which makes the results
 * bit-identical to an AVX2+FMA build of the reference compiled with
 * -ffp-contract=off.
 */
#pragma once
#include <stdint.h>
#ifndef EK_HOST_EMU
#include <cuda_runtime.h>
#endif

namespace ekm {

__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float fbits(uint32_t u) { return __uint_as_float(u); }
__device__ __forceinline__ uint32_t ubits(float f) { return __float_as_uint(f); }

/* x86 cvttps2dq semantics: out-of-range and NaN give the "integer indefinite" 0x80000000 */
__device__ __forceinline__ int32_t cvtt_f32_i32(float x) {
    return (x >= -2147483648.f && x < 2147483648.f) ? __float2int_rz(x) : (int32_t) 0x80000000;
}
/* Saturating conversion (cvt.rzi.s32.f32) where the difference to cvttps2dq cannot be observed:
   - sincos: the argument is >= 0; positive overflow saturates to 0x7fffffff and (j + 1) & ~1 maps it to the
     same 0x80000000 the CPU path produces; NaN ends in NaN either way;
   - exp: the argument is an integer in [-128, 128] unless the overflow/underflow masks or a NaN override it. */
__device__ __forceinline__ int32_t cvtt_sat(float x) { return __float2int_rz(x); }

/* array_math.h:25-33 */
__device__ __forceinline__ float poly2(float x, float c0, float c1, float c2) {
    float x2 = fmul(x, x);
    return ffma(x2, c2, ffma(x, c1, c0));
}
/* array_math.h:50-58 */
__device__ __forceinline__ float poly5(float x, float c0, float c1, float c2, float c3, float c4, float c5) {
    float x2 = fmul(x, x), x4 = fmul(x2, x2);
    return ffma(x2, ffma(x, c3, c2), ffma(x4, ffma(x, c5, c4), ffma(x, c1, c0)));
}
/* array_math.h:80-88 */
__device__ __forceinline__ float poly8(float x, float c0, float c1, float c2, float c3, float c4,
                                       float c5, float c6, float c7, float c8) {
    float x2 = fmul(x, x), x4 = fmul(x2, x2), x8 = fmul(x4, x4);
    return ffma(x4, ffma(x2, ffma(x, c7, c6), ffma(x, c5, c4)),
                ffma(x2, ffma(x, c3, c2), fadd(ffma(x, c1, c0), fmul(c8, x8))));
}

/* array_math.h:261-367 sincos_approx<Sin, Cos>, single precision branch */
template <bool Sin, bool Cos>
__device__ __forceinline__ void sincos(float x, float &s_out, float &c_out) {
    float xa = fabsf(x);
    int32_t j = cvtt_sat(fmul(xa, 1.2732395447351626862f));
    j = (j + 1) & ~1;
    float y = __int2float_rn(j);
    uint32_t sign_sin = ((uint32_t) j << 29) ^ ubits(x);
    uint32_t sign_cos = (uint32_t) (~(j - 2)) << 29;
    y = fsub(fsub(fsub(xa, fmul(y, 0.78515625f)), fmul(y, 2.4187564849853515625e-4f)),
             fmul(y, 3.77489497744594108e-8f));
    float z = fmul(y, y);
    if (xa == __int_as_float(0x7f800000)) z = fbits(0xffffffffu);
    float s = fmul(poly2(z, -1.6666654611e-1f, 8.3321608736e-3f, -1.9515295891e-4f), z);
    float c = fmul(poly2(z, 4.166664568298827e-2f, -1.388731625493765e-3f, 2.443315711809948e-5f), z);
    s = ffma(s, y, y);
    c = ffma(c, z, ffma(z, -0.5f, 1.f));
    bool polymask = (j & 2) == 0;
    if (Sin) s_out = fbits(ubits(polymask ? s : c) ^ (sign_sin & 0x80000000u));
    if (Cos) c_out = fbits(ubits(polymask ? c : s) ^ (sign_cos & 0x80000000u));
}
__device__ __forceinline__ float sin_f32(float x) { float s, c; sincos<true, false>(x, s, c); return s; }
__device__ __forceinline__ float cos_f32(float x) { float s, c; sincos<false, true>(x, s, c); return c; }

/* array_math.h:711-776 exp, single precision branch (+ ldexp :677-680) */
__device__ __forceinline__ float exp_f32(float x) {
    const float max_range = +88.3762588501f, min_range = -88.3762588501f;
    bool overflow = x > max_range, underflow = x < min_range;
    float n = floorf(ffma(1.4426950408889634073599f, x, 0.5f));
    float xr = ffma(-n, 0.693359375f, x);
    xr = ffma(-n, -2.12194440e-4f, xr);
    float z = poly5(xr, 5.0000001201e-1f, 1.6666665459e-1f, 4.1665795894e-2f,
                        8.3334519073e-3f, 1.3981999507e-3f, 1.9875691500e-4f);
    z = ffma(z, fmul(xr, xr), fadd(xr, 1.f));
    uint32_t scale = (uint32_t) (cvtt_sat(n) + 0x7f) << 23;
    float r = fmul(z, fbits(scale));
    return overflow ? __int_as_float(0x7f800000) : (underflow ? 0.f : r);
}

/* array_math.h:778-898 log, single precision branch, non-AVX512 (frexp :682-709) */
__device__ __forceinline__ float log_f32(float x) {
    bool valid = x >= 0.f;
    uint32_t xi = ubits(x);
    uint32_t exponent_bits = xi & 0x7f800000u;
    bool is_normal = (x != 0.f) && (exponent_bits != 0x7f800000u);
    int32_t exponent_i = (int32_t) (exponent_bits >> 23) - 0x7f;
    uint32_t mantissa = (xi & ~0x7f800000u) | 0x3f000000u;
    float xm = fbits(is_normal ? mantissa : xi);
    float e = __int2float_rn(is_normal ? exponent_i : 0);

    bool ge = xm >= 0.70710678118654752440f;
    if (ge) e = fadd(e, 1.f);
    xm = fadd(xm, fsub(ge ? 0.f : xm, 1.f));

    float z = fmul(xm, xm);
    float y = poly8(xm, 3.3333331174e-1f, -2.4999993993e-1f, 2.0000714765e-1f, -1.6668057665e-1f,
                        1.4249322787e-1f, -1.2420140846e-1f, 1.1676998740e-1f, -1.1514610310e-1f,
                        7.0376836292e-2f);
    y = fmul(y, fmul(xm, z));
    y = ffma(e, -2.12194440e-4f, y);
    z = ffma(z, -0.5f, fadd(xm, y));
    float r = ffma(e, 0.693359375f, z);
    if (x == __int_as_float(0x7f800000)) r = __int_as_float(0x7f800000);
    if (x == 0.f) r = __int_as_float(0xff800000);
    return valid ? r : fbits(0xffffffffu);
}

/* ---------------- tan, cot, asin, acos, atan, atan2 ----------------
   The single precision branches of array_math.h, restated operation for operation as the reference's generic body
   records them on this backend (one node per primitive): separate mul / sub roundings, the same fmadd Estrin groupings,
   cvttps2dq truncation, select, bit operations, and the correctly rounded rcp / division of DESIGN.md §4.  A result
   is therefore bit-identical to the traced form, NaNs included.  Constants that the reference writes as double
   literals are rounded to float once, as Scalar(c) does. */

/* min/max with the x86 vminps/vmaxps operand rule of the CPU path
   (array_avx.h min_/max_: second operand returned when either is NaN) */
__device__ __forceinline__ float min_x86(float a, float b) { return a < b ? a : b; }
__device__ __forceinline__ float max_x86(float a, float b) { return a > b ? a : b; }

/* array_math.h:39-45 */
__device__ __forceinline__ float poly4(float x, float c0, float c1, float c2, float c3, float c4) {
    float x2 = fmul(x, x), x4 = fmul(x2, x2);
    return ffma(x2, ffma(x, c3, c2), fadd(ffma(x, c1, c0), fmul(c4, x4)));
}
/* array_math.h:56-63 */
__device__ __forceinline__ float poly6(float x, float c0, float c1, float c2, float c3, float c4, float c5, float c6) {
    float x2 = fmul(x, x), x4 = fmul(x2, x2);
    return ffma(x4, ffma(x2, c6, ffma(x, c5, c4)), ffma(x2, ffma(x, c3, c2), ffma(x, c1, c0)));
}

/* array_math.h:369-442 tancot_approx<Tan>, single precision branch (tan :466-468, cot :470-472) */
template <bool Tan>
__device__ __forceinline__ float tancot_f32(float x) {
    float xa = fabsf(x);
    int32_t j = cvtt_f32_i32(fmul(xa, (float) 1.2732395447351626862));
    j = (j + 1) & ~1;
    float y = __int2float_rn(j);
    y = fsub(fsub(fsub(xa, fmul(y, (float) 0.78515625)), fmul(y, (float) 2.4187564849853515625e-4)),
             fmul(y, (float) 3.77489497744594108e-8));
    float z = fmul(y, y);
    if (xa == __int_as_float(0x7f800000)) z = fbits(0xffffffffu);         /* z |= eq(xa, inf) */
    float r = poly5(z, (float) 3.33331568548e-1, (float) 1.33387994085e-1, (float) 5.34112807005e-2,
                       (float) 2.44301354525e-2, (float) 3.11992232697e-3, (float) 9.38540185543e-3);
    r = ffma(r, fmul(z, y), y);
    if (xa < (float) 1e-4) r = y;
    const bool recip = Tan ? (j & 2) != 0 : (j & 2) == 0;
    if (recip) r = __frcp_rn(r);
    return fbits(ubits(r) ^ ((((uint32_t) j << 30) ^ ubits(x)) & 0x80000000u));   /* mulsign(r, sign) */
}
__device__ __forceinline__ float tan_f32(float x) { return tancot_f32<true>(x); }
__device__ __forceinline__ float cot_f32(float x) { return tancot_f32<false>(x); }

/* the shared part of array_math.h:493-508 (asin) and :570-585 (acos): returns z1, sets big = |x| > 0.5 */
__device__ __forceinline__ float asincos_core(float x, float c0, bool &big) {
    float xa = fabsf(x), x2 = fmul(x, x);
    big = xa > 0.5f;
    float x1 = fmul(0.5f, fsub(1.f, xa));
    float x3 = big ? x1 : x2;
    float x4 = big ? __fsqrt_rn(x1) : xa;
    float z1 = poly4(x3, c0, 7.4953002686e-2f, 4.5470025998e-2f, 2.4181311049e-2f, 4.2163199048e-2f);
    return ffma(z1, fmul(x3, x4), x4);
}
/* array_math.h:474-553 asin, single precision branch; copysign(r, x) = |r| | (x & sign) (array_router.h:398) */
__device__ __forceinline__ float asin_f32(float x) {
    bool big;
    float z1 = asincos_core(x, 1.6666752422e-1f, big);
    float r = big ? fsub((float) 1.57079632679489661923, fadd(z1, z1)) : z1;
    return fbits((ubits(r) & 0x7fffffffu) | (ubits(x) & 0x80000000u));
}
/* array_math.h:555-590 acos, single precision branch */
__device__ __forceinline__ float acos_f32(float x) {
    bool big;
    float z1 = asincos_core(x, 1.666675242e-1f, big);
    float z2 = fadd(z1, z1);
    if (x < 0.f) z2 = fsub((float) 3.14159265358979323846, z2);
    float z3 = fsub((float) 1.57079632679489661923, fbits((ubits(z1) & 0x7fffffffu) | (ubits(x) & 0x80000000u)));
    return big ? z2 : z3;
}
/* array_math.h:603-664 atan2(y, x), single precision branch.  min / max are the backend's (x86 operand rule),
   1 / max is a correctly rounded division, and r &= neq(max, 0) selects +0. */
__device__ __forceinline__ float atan2_f32(float y, float x) {
    float abs_x = fabsf(x), abs_y = fabsf(y);
    float min_val = min_x86(abs_y, abs_x), max_val = max_x86(abs_x, abs_y);
    float scaled_min = fmul(min_val, __fdiv_rn(1.f, max_val));
    float z = fmul(scaled_min, scaled_min);
    float t = poly6(z, (float) 0.99999934166683966009, (float) -0.33326497518773606976, (float) +0.19881342388439013552,
                       (float) -0.13486708938456973185, (float) +0.083863120428809689910, (float) -0.037006525670417265220,
                       (float) 0.0078613793713198150252);
    t = fmul(t, scaled_min);
    if (abs_y > abs_x) t = fsub((float) 1.57079632679489661923, t);
    if (x < 0.f) t = fsub((float) 3.14159265358979323846, t);
    float r = y < 0.f ? fbits(ubits(t) ^ 0x80000000u) : t;
    return max_val != 0.f ? r : 0.f;
}
/* array_math.h:666-668: atan(x) = atan2(x, 1) */
__device__ __forceinline__ float atan_f32(float x) { return atan2_f32(x, 1.f); }

/* ---------------- sinh, cosh, tanh, asinh, acosh, atanh, cbrt ----------------
   Restated like the trigonometric functions above: each is the operation sequence of the traced single precision body,
   with this backend's exp_f32 / log_f32, the correctly rounded rcp, sqrt and division, and the mask operations as the
   bit operations the backend records for them: value & ~mask gives +0 where the mask is set, value | mask all ones. */

/* array_math.h:31-37 */
__device__ __forceinline__ float poly3(float x, float c0, float c1, float c2, float c3) {
    float x2 = fmul(x, x);
    return ffma(x2, ffma(x, c3, c2), ffma(x, c1, c0));
}
/* copysign(r, x) = |r| | (x & sign) (array_router.h:398) */
__device__ __forceinline__ float copysign_bits(float r, float x) {
    return fbits((ubits(r) & 0x7fffffffu) | (ubits(x) & 0x80000000u));
}

/* array_math.h:1067-1127 sincosh, which is sinh :997-1046 and cosh :1048-1065 computed together: both start from
   exp0 = exp(x), exp1 = rcp(exp0) */
template <bool Sinh, bool Cosh>
__device__ __forceinline__ void sincosh_f32(float x, float &s_out, float &c_out) {
    float exp0 = exp_f32(x), exp1 = __frcp_rn(exp0);
    if (Sinh) {
        float x2 = fmul(x, x);
        float r_small = ffma(poly2(x2, (float) 1.66667160211e-1, (float) 8.33028376239e-3, (float) 2.03721912945e-4),
                             fmul(x2, x), x);
        float r_big = fmul(fsub(exp0, exp1), 0.5f);
        s_out = fabsf(x) > 1.f ? r_big : r_small;
    }
    if (Cosh) c_out = fmul(fadd(exp0, exp1), 0.5f);
}
__device__ __forceinline__ float sinh_f32(float x) { float s, c; sincosh_f32<true, false>(x, s, c); return s; }
__device__ __forceinline__ float cosh_f32(float x) { float s, c; sincosh_f32<false, true>(x, s, c); return c; }

/* array_math.h:1129-1179 tanh, single precision branch */
__device__ __forceinline__ float tanh_f32(float x) {
    float x2 = fmul(x, x);
    float r_small = poly4(x2, (float) -3.33332819422e-1, (float) 1.33314422036e-1, (float) -5.37397155531e-2,
                              (float) 2.06390887954e-2, (float) -5.70498872745e-3);
    r_small = ffma(r_small, fmul(x2, x), x);
    float e = exp_f32(fadd(x, x)), e2 = __frcp_rn(fadd(e, 1.f));
    float r_big = fsub(1.f, fadd(e2, e2));
    return fabsf(x) >= 0.625f ? r_big : r_small;
}

/* array_math.h:1185-1237 asinh, single precision branch */
__device__ __forceinline__ float asinh_f32(float x) {
    float x2 = fmul(x, x), xa = fabsf(x);
    bool big = xa >= (float) 0.51, huge = xa >= (float) 1e10;
    float r_small = poly3(x2, (float) -1.6666288134e-1, (float) 7.4847586088e-2, (float) -4.2699340972e-2,
                              (float) 2.0122003309e-2);
    r_small = ffma(r_small, fmul(x2, x), x);
    float r_big = log_f32(fadd(huge ? 0.f : __fsqrt_rn(fadd(x2, 1.f)), xa));     /* sqrt(x2 + 1) & ~mask_huge */
    if (huge) r_big = fadd(r_big, (float) 0.693147180559945309417);               /* r_big[mask_huge] += M_LN2 */
    r_big = copysign_bits(r_big, x);
    return big ? r_big : r_small;
}

/* array_math.h:1239-1293 acosh, single precision branch.  fmsub(x, x, 1) is fma(x, x, -1). */
__device__ __forceinline__ float acosh_f32(float x) {
    float x1 = fsub(x, 1.f);
    bool big = x1 >= (float) 0.49, huge = x1 >= (float) 1e10;
    float r_small = poly4(x1, (float) 1.4142135263e+0, (float) -1.1784741703e-1, (float) 2.6454905019e-2,
                              (float) -7.5272886713e-3, (float) 1.7596881071e-3);
    r_small = fmul(__fsqrt_rn(x1), r_small);
    if (x1 < 0.f) r_small = fbits(0xffffffffu);                                   /* r_small |= x1 < 0 */
    float r_big = log_f32(fadd(huge ? 0.f : __fsqrt_rn(ffma(x, x, -1.f)), x));
    if (huge) r_big = fadd(r_big, (float) 0.693147180559945309417);
    return big ? r_big : r_small;
}

/* array_math.h:1295-1348 atanh, single precision branch */
__device__ __forceinline__ float atanh_f32(float x) {
    float xa = fabsf(x), x2 = fmul(x, x);
    float r_small = poly4(x2, (float) 3.33337300303e-1, (float) 1.99782164500e-1, (float) 1.46691431730e-1,
                              (float) 8.24370301058e-2, (float) 1.81740078349e-1);
    r_small = ffma(r_small, fmul(x2, x), x);
    float r_big = fmul(log_f32(__fdiv_rn(fadd(xa, 1.f), fsub(1.f, xa))), 0.5f);
    r_big = copysign_bits(r_big, x);
    return xa >= 0.5f ? r_big : r_small;
}

/* array_math.h:900-954 cbrt, single precision branch (one Newton step), with frexp :682-709 and ldexp :677-680.  frexp
   treats 0 and denormals as normal numbers: cbrt(+-0) is +-0.337986261 and cbrt(1e-45) 1.2e-13, as on the CPU path. */
__device__ __forceinline__ float cbrt_f32(float x) {
    const float third = (float) (1.0 / 3.0);
    float xa = fabsf(x);
    uint32_t xi = ubits(xa), exponent_bits = xi & 0x7f800000u;
    bool is_normal = exponent_bits != 0x7f800000u && xa != 0.f;
    float xm = fbits(is_normal ? (xi & 0x807fffffu) | 0x3f000000u : xi);
    float xe = fadd(__int2float_rn(is_normal ? (int32_t) (exponent_bits >> 23) - 0x7f : 0), 1.f);
    float xea = fabsf(xe), xea1 = floorf(fmul(xea, third));
    float rem = ffma(xea1, -3.f, xea);                                            /* fnmadd(xea1, 3, xea) */
    xm = poly4(xm, (float) 0.40238979564544752126924, (float) 1.1399983354717293273738,
                   (float) -0.95438224771509446525043, (float) 0.54664601366395524503440,
                   (float) -0.13466110473359520655053);
    /* CBRT2, CBRT4 and Scalar(1) / CBRT2, Scalar(1) / CBRT4, the latter two divided in float */
    float f1 = xe >= 0.f ? fbits(0x3fa14518u) : fbits(0x3f4b2ff5u);
    float f2 = xe >= 0.f ? fbits(0x3fcb2ff5u) : fbits(0x3f214518u);
    float f = rem == 1.f ? f1 : f2;
    if (rem != 0.f) xm = fmul(f, xm);                                             /* xm[neq(rem, 0)] *= f */
    float e = fbits(ubits(xea1) ^ (ubits(xe) & 0x80000000u));                     /* mulsign(xea1, xe) */
    float r = fmul(fbits(((uint32_t) cvtt_f32_i32(e) + 0x7fu) << 23), xm);        /* ldexp(xm, e) */
    r = fbits(ubits(r) ^ (ubits(x) & 0x80000000u));                               /* mulsign(r, x) */
    r = fsub(r, fmul(fsub(r, __fdiv_rn(x, fmul(r, r))), third));
    return fabsf(x) < __int_as_float(0x7f800000) ? r : x;
}

/* ---------------- erf, erfc, erfinv, lgamma, tgamma ----------------
   The single precision branches of special.h, restated the same way: the operation sequence that the generic body
   records on this backend, with this backend's exp_f32 / log_f32 / sin_f32, the correctly rounded rcp and division,
   rintf for round (ROUND_F32), negation as a sign flip (NEG_F32) and the coefficients rounded to float as Scalar(c)
   rounds them.  On a CUDA array both sides of every branch are recorded and selected; evaluating only the selected
   side gives the same bits. */

/* array_math.h:65-72 */
__device__ __forceinline__ float poly7(float x, float c0, float c1, float c2, float c3, float c4, float c5, float c6,
                                       float c7) {
    float x2 = fmul(x, x), x4 = fmul(x2, x2);
    return ffma(x4, ffma(x2, ffma(x, c7, c6), ffma(x, c5, c4)), ffma(x2, ffma(x, c3, c2), ffma(x, c1, c0)));
}
__device__ __forceinline__ float fneg(float x) { return fbits(ubits(x) ^ 0x80000000u); }

/* special.h:56-129 erfc<T, false>, single precision branch (the body without its |x| < 1 recursion into erf) */
__device__ __forceinline__ float erfc_core_f32(float x) {
    float xa = fabsf(x), q = __frcp_rn(xa), y = fmul(q, q);
    float p_small = poly8(y, (float) 5.638259427386472e-1, (float) -2.741127028184656e-1, (float) 3.404879937665872e-1,
                             (float) -4.944515323274145e-1, (float) 6.210004621745983e-1, (float) -5.824733027278666e-1,
                             (float) 3.687424674597105e-1, (float) -1.387039388740657e-1, (float) 2.326819970068386e-2);
    float p_large = poly7(y, (float) 5.641895067754075e-1, (float) -2.820767439740514e-1, (float) 4.218463358204948e-1,
                             (float) -1.015265279202700e+0, (float) 2.921019019210786e+0, (float) -7.495518717768503e+0,
                             (float) 1.297719955372516e+1, (float) -1.047766399936249e+1);
    float r = fmul(fmul(exp_f32(fmul(fneg(x), x)), q), xa > 2.f ? p_large : p_small);
    return x < 0.f ? fsub(2.f, r) : r;                                            /* r[x < 0] = 2 - r */
}
/* special.h:131-164 erf<T, false>, single precision branch (the body without its |x| > 1 recursion into erfc) */
__device__ __forceinline__ float erf_core_f32(float x) {
    float r = poly6(fmul(x, x), (float) 1.128379165726710e+0, (float) -3.761262582423300e-1,
                                (float) 1.128358514861418e-1, (float) -2.685381193529856e-2,
                                (float) 5.188327685732524e-3, (float) -8.010193625184903e-4,
                                (float) 7.853861353153693e-5);
    return fmul(r, x);
}
/* special.h:131-164 erf: r[|x| > 1] = 1 - erfc<T, false>(x) */
__device__ __forceinline__ float erf_f32(float x) {
    return fabsf(x) > 1.f ? fsub(1.f, erfc_core_f32(x)) : erf_core_f32(x);
}
/* special.h:56-129 erfc: r[|x| < 1] = 1 - erf<T, false>(x).  At |x| == 1 erf takes its polynomial and erfc its own
   formula. */
__device__ __forceinline__ float erfc_f32(float x) {
    return fabsf(x) < 1.f ? fsub(1.f, erf_core_f32(x)) : erfc_core_f32(x);
}

/* special.h:222-246 erfinv */
__device__ __forceinline__ float erfinv_f32(float x) {
    float w = fneg(log_f32(fmul(fadd(1.f, x), fsub(1.f, x))));
    float w1 = fsub(w, 2.5f), w2 = fsub(__fsqrt_rn(w), 3.f);
    float p1 = poly8(w1, (float) 1.50140941, (float) 0.246640727, (float) -0.00417768164, (float) -0.00125372503,
                         (float) 0.00021858087, (float) -4.39150654e-06, (float) -3.5233877e-06, (float) 3.43273939e-07,
                         (float) 2.81022636e-08);
    float p2 = poly8(w2, (float) 2.83297682, (float) 1.00167406, (float) 0.00943887047, (float) -0.0076224613,
                         (float) 0.00573950773, (float) -0.00367342844, (float) 0.00134934322, (float) 0.000100950558,
                         (float) -0.000200214257);
    return fmul(w < 5.f ? p1 : p2, x);
}

/* special.h:275-309 lgamma (Lanczos, g = 5, n = 6).  The sum starts from a recorded literal 0, so a -0 quotient becomes
   +0; b = (x + 5) + 0.5 rounds twice. */
__device__ __forceinline__ float lgamma_f32(float x_) {
    const float pi = (float) 3.14159265358979323846;
    bool reflect = x_ < 0.5f;
    float x = reflect ? fneg(x_) : fsub(x_, 1.f);
    float sum = fadd(__fdiv_rn((float) -0.5395239384953e-5, fadd(x, 6.f)), 0.f);
    sum = fadd(sum, __fdiv_rn((float) 0.1208650973866179e-2, fadd(x, 5.f)));
    sum = fadd(sum, __fdiv_rn((float) -1.231739572450155, fadd(x, 4.f)));
    sum = fadd(sum, __fdiv_rn((float) 24.01409824083091, fadd(x, 3.f)));
    sum = fadd(sum, __fdiv_rn((float) -86.50532032941677, fadd(x, 2.f)));
    sum = fadd(sum, __fdiv_rn((float) 76.18009172947146, fadd(x, 1.f)));
    sum = fadd(sum, (float) 1.000000000190015);
    float b = fadd(fadd(x, 5.f), 0.5f);
    float result = fadd(fsub(fadd((float) 0.91893853320467274178, log_f32(sum)), b), fmul(log_f32(b), fadd(x, 0.5f)));
    if (reflect) {
        result = fsub(log_f32(fabsf(__fdiv_rn(pi, sin_f32(fmul(pi, x_))))), result);
        if (x_ == rintf(x_)) result = __int_as_float(0x7f800000);
    }
    return result;
}
/* special.h:312 tgamma = exp(lgamma(x)) */
__device__ __forceinline__ float tgamma_f32(float x) { return exp_f32(lgamma_f32(x)); }

/* ---------------- pow, frexp, hypot, dawson, erfi ----------------
   Further single precision bodies of array_math.h and special.h, restated the same way: this backend's exp_f32 /
   log_f32, the correctly rounded division and sqrt, min / max with the x86 operand rule, and the coefficients rounded to
   float as Scalar(c) rounds them. */

/* array_math.h:956-958 pow = exp(log(x) * y): pow(0, 0) = exp(-inf * 0) is NaN, as is the power of a negative base */
__device__ __forceinline__ float pow_f32(float x, float y) { return exp_f32(fmul(log_f32(x), y)); }

/* array_math.h:682-709 frexp: (mantissa | 0.5, biased exponent - 0x7f) for every number whose exponent field is not all
   ones except +-0, denormals included (their mantissa keeps its leading zeros, their exponent is -127); (x, 0) for
   +-0, +-inf and NaN */
__device__ __forceinline__ bool frexp_normal(float x) { return x != 0.f && (ubits(x) & 0x7f800000u) != 0x7f800000u; }
__device__ __forceinline__ float frexp_m_f32(float x) {
    return frexp_normal(x) ? fbits((ubits(x) & ~0x7f800000u) | 0x3f000000u) : x;
}
__device__ __forceinline__ float frexp_e_f32(float x) {
    return __int2float_rn(frexp_normal(x) ? (int32_t) ((ubits(x) & 0x7f800000u) >> 23) - 0x7f : 0);
}

/* array_math.h:1362-1379 hypot: max * sqrt(1 + (min / max)^2) where both operands and the ratio are finite, |a| + |b|
   elsewhere */
__device__ __forceinline__ float hypot_f32(float a, float b) {
    const float inf = __int_as_float(0x7f800000);
    float abs_a = fabsf(a), abs_b = fabsf(b);
    float maxval = max_x86(abs_a, abs_b), minval = min_x86(abs_a, abs_b), ratio = __fdiv_rn(minval, maxval);
    return abs_a < inf && abs_b < inf && ratio < inf ? fmul(maxval, __fsqrt_rn(fadd(1.f, fmul(ratio, ratio))))
                                                     : fadd(abs_a, abs_b);
}

/* special.h:249-265 dawson = num(x^2) / denom(x^2) * x */
__device__ __forceinline__ float dawson_f32(float x) {
    float x2 = fmul(x, x);
    float num = poly6(x2, (float) 1.00000080272429, (float) 9.18170212243285e-2, (float) 4.25835373536124e-2,
                          (float) 6.0536496345054e-3, (float) 9.88555033724111e-4, (float) 3.64943550840577e-5,
                          (float) 1.55942290996993e-5);
    float denom = poly7(x2, 1.f, (float) 7.58517175815194e-1, (float) 2.81364355593059e-1, (float) 6.81783097841267e-2,
                            (float) 1.13586116798019e-2, (float) 1.92020805811771e-3, (float) 5.74217664074868e-5,
                            (float) 3.11884331363595e-5);
    return fmul(__fdiv_rn(num, denom), x);
}

/* special.h:267-271 erfi = M_2_SQRTPI * dawson(x) * exp(x * x) */
__device__ __forceinline__ float erfi_f32(float x) {
    return fmul(fmul((float) 1.12837916709551257390, dawson_f32(x)), exp_f32(fmul(x, x)));
}

/* ---------------- carlson_rf, carlson_rd, carlson_rc ----------------
   The single precision bodies of special.h's Carlson integrals, one element at a time.  special.h runs their
   duplication loop on the host over whole arrays: every update is masked by `active`, which only ever turns off, and the
   loop ends when no element is active or after the tenth evaluation of the loop head.  An element that has stopped keeps
   its arguments, so each later pass recomputes the same XYZ and mu_inv for it; element by element the loop is therefore
   "evaluate the head; stop if !(eps > threshold) or this was the tenth head; update", which is what these loops do.
   The operations are the recorded ones: correctly rounded sqrt, rcp and division; dot() of a nested array as
   array_static.h:948-958's product and fmadd chain; hsum / hprod / hmax as left folds, hmax with the x86 max rule;
   fnmadd as one fma; masked updates as selects; constants and thresholds rounded to float as Scalar(c) rounds them. */

/* special.h:325-366 carlson_rf(x, y, z) */
__device__ __forceinline__ float carlson_rf_f32(float x, float y, float z) {
    const float thr = (float) 0.070154;
    float X, Y, Z, mu_inv;
#pragma unroll 1
    for (int it = 1;; ++it) {
        const float sx = __fsqrt_rn(x), sy = __fsqrt_rn(y), sz = __fsqrt_rn(z);
        const float lambda = ffma(sx, sz, ffma(sz, sy, fmul(sy, sx)));          /* dot(shuffle<1, 2, 0>(s), s) */
        const float mu = fmul(fadd(fadd(x, y), z), (float) (1.0 / 3.0));
        mu_inv = __frcp_rn(mu);
        X = ffma(-x, mu_inv, 1.f); Y = ffma(-y, mu_inv, 1.f); Z = ffma(-z, mu_inv, 1.f);
        const float eps = max_x86(max_x86(fabsf(X), fabsf(Y)), fabsf(Z));
        if (!(eps > thr) || it == 10) break;
        x = fmul(fadd(x, lambda), 0.25f); y = fmul(fadd(y, lambda), 0.25f); z = fmul(fadd(z, lambda), 0.25f);
    }
    const float e2 = fsub(fmul(X, Y), fmul(Z, Z)), e3 = fmul(fmul(X, Y), Z);
    const float er = fadd(fmul(fsub(fsub(fmul((float) (1.0 / 24.0), e2), (float) (1.0 / 10.0)),
                                    fmul((float) (3.0 / 44.0), e3)), e2),
                          fmul((float) (1.0 / 14.0), e3));
    return fmul(__fsqrt_rn(mu_inv), fadd(1.f, er));
}

/* special.h:379-432 carlson_rd(x, y, z) */
__device__ __forceinline__ float carlson_rd_f32(float x, float y, float z) {
    const float thr = (float) (0.070154 * 0.6);
    const float w0 = (float) (1.0 / 5.0), w2 = (float) (3.0 / 5.0);
    float X, Y, Z, mu_inv, sum = 0.f, num = 1.f;
#pragma unroll 1
    for (int it = 1;; ++it) {
        const float sx = __fsqrt_rn(x), sy = __fsqrt_rn(y), sz = __fsqrt_rn(z);
        const float lambda = ffma(sx, sz, ffma(sz, sy, fmul(sy, sx)));
        const float mu = fadd(fadd(fmul(x, w0), fmul(y, w0)), fmul(z, w2));     /* hsum(xyz * W) */
        mu_inv = __frcp_rn(mu);
        X = ffma(-x, mu_inv, 1.f); Y = ffma(-y, mu_inv, 1.f); Z = ffma(-z, mu_inv, 1.f);
        const float eps = max_x86(max_x86(fabsf(X), fabsf(Y)), fabsf(Z));
        if (!(eps > thr) || it == 10) break;
        sum = fadd(sum, __fdiv_rn(num, fmul(sz, fadd(z, lambda))));
        num = fmul(num, 0.25f);
        x = fmul(fadd(x, lambda), 0.25f); y = fmul(fadd(y, lambda), 0.25f); z = fmul(fadd(z, lambda), 0.25f);
    }
    const float ea = fmul(X, Y), eb = fmul(Z, Z), ec = fsub(ea, eb);
    const float ed = ffma(-6.f, eb, ea), ee = ffma(ec, 2.f, ed);
    const float p1 = fmul(ed, fsub(fadd(-(float) (3.0 / 14.0), fmul((float) (9.0 / 88.0), ed)),
                                   fmul(fmul(0.25f, Z), ee)));
    const float p2 = fmul(Z, fadd(fmul((float) (1.0 / 6.0), ee),
                                  fmul(Z, fadd(fmul(-(float) (9.0 / 22.0), ec), fmul(fmul(Z, (float) (3.0 / 26.0)), ea)))));
    const float p = fadd(p1, p2);
    return fadd(fmul(3.f, sum), fmul(fmul(fmul(num, mu_inv), __fsqrt_rn(mu_inv)), fadd(1.f, p)));
}

/* special.h:445-482 carlson_rc(x, y); lambda += lambda + y rounds twice */
__device__ __forceinline__ float carlson_rc_f32(float x, float y) {
    const float thr = (float) (0.070154 * 0.48);
    float inv_mu, s;
#pragma unroll 1
    for (int it = 1;; ++it) {
        float lambda = fmul(__fsqrt_rn(x), __fsqrt_rn(y));
        lambda = fadd(lambda, fadd(lambda, y));
        const float mu = ffma(x, (float) (1.0 / 3.0), fmul(y, (float) (2.0 / 3.0)));
        inv_mu = __frcp_rn(mu);
        s = fmul(fsub(y, mu), inv_mu);
        if (!(fabsf(s) > thr) || it == 10) break;
        x = fmul(fadd(x, lambda), 0.25f); y = fmul(fadd(y, lambda), 0.25f);
    }
    const float q = fadd(0.3f, fmul(s, fadd((float) (1.0 / 7.0), fmul(s, fadd(0.375f, fmul(s, (float) (9.0 / 22.0)))))));
    return fmul(__fsqrt_rn(inv_mu), fadd(1.f, fmul(fmul(s, s), q)));
}

/* ---------------- two elements at a time ----------------
   The sweep kernels evaluate exp / sin / cos on pairs of elements: the two independent dependency chains give
   ptxas instruction-level parallelism to interleave.  sm_90 has no packed fp32 arithmetic, so every pair
   operation is two scalar IEEE operations, rounded exactly like the scalar code above. */
struct f2 { float x, y; };
__device__ __forceinline__ f2 mk2(float v) { return f2{ v, v }; }
__device__ __forceinline__ f2 ffma2(f2 a, f2 b, f2 c) { return f2{ ffma(a.x, b.x, c.x), ffma(a.y, b.y, c.y) }; }
__device__ __forceinline__ f2 fmul2(f2 a, f2 b) { return f2{ fmul(a.x, b.x), fmul(a.y, b.y) }; }
__device__ __forceinline__ f2 fadd2(f2 a, f2 b) { return f2{ fadd(a.x, b.x), fadd(a.y, b.y) }; }
__device__ __forceinline__ f2 fsub2(f2 a, f2 b) { return f2{ fsub(a.x, b.x), fsub(a.y, b.y) }; }
__device__ __forceinline__ f2 ffma2(f2 a, float b, float c) { return ffma2(a, mk2(b), mk2(c)); }
__device__ __forceinline__ f2 ffma2(f2 a, float b, f2 c) { return ffma2(a, mk2(b), c); }
__device__ __forceinline__ f2 fmul2(f2 a, float b) { return fmul2(a, mk2(b)); }

__device__ __forceinline__ f2 poly2(f2 x, float c0, float c1, float c2) {
    f2 x2 = fmul2(x, x);
    return ffma2(x2, c2, ffma2(x, c1, c0));
}
__device__ __forceinline__ f2 poly5(f2 x, float c0, float c1, float c2, float c3, float c4, float c5) {
    f2 x2 = fmul2(x, x), x4 = fmul2(x2, x2);
    return ffma2(x2, ffma2(x, c3, c2), ffma2(x4, ffma2(x, c5, c4), ffma2(x, c1, c0)));
}
/* two elements of sincos_approx (same steps as sincos<> above) */
template <bool Sin, bool Cos>
__device__ __forceinline__ void sincos2(f2 x, f2 &s_out, f2 &c_out) {
    f2 xa = { fabsf(x.x), fabsf(x.y) };
    f2 q = fmul2(xa, 1.2732395447351626862f);
    int32_t j0 = (cvtt_sat(q.x) + 1) & ~1, j1 = (cvtt_sat(q.y) + 1) & ~1;
    f2 y = { __int2float_rn(j0), __int2float_rn(j1) };
    y = fsub2(fsub2(fsub2(xa, fmul2(y, 0.78515625f)), fmul2(y, 2.4187564849853515625e-4f)),
              fmul2(y, 3.77489497744594108e-8f));
    f2 z = fmul2(y, y);
    if (xa.x == __int_as_float(0x7f800000)) z.x = fbits(0xffffffffu);
    if (xa.y == __int_as_float(0x7f800000)) z.y = fbits(0xffffffffu);
    f2 s = fmul2(poly2(z, -1.6666654611e-1f, 8.3321608736e-3f, -1.9515295891e-4f), z);
    f2 c = fmul2(poly2(z, 4.166664568298827e-2f, -1.388731625493765e-3f, 2.443315711809948e-5f), z);
    s = ffma2(s, y, y);
    c = ffma2(c, z, ffma2(z, -0.5f, 1.f));
    bool p0 = (j0 & 2) == 0, p1 = (j1 & 2) == 0;
    if (Sin) {
        s_out.x = fbits(ubits(p0 ? s.x : c.x) ^ ((((uint32_t) j0 << 29) ^ ubits(x.x)) & 0x80000000u));
        s_out.y = fbits(ubits(p1 ? s.y : c.y) ^ ((((uint32_t) j1 << 29) ^ ubits(x.y)) & 0x80000000u));
    }
    if (Cos) {
        c_out.x = fbits(ubits(p0 ? c.x : s.x) ^ (((uint32_t) (~(j0 - 2)) << 29) & 0x80000000u));
        c_out.y = fbits(ubits(p1 ? c.y : s.y) ^ (((uint32_t) (~(j1 - 2)) << 29) & 0x80000000u));
    }
}
__device__ __forceinline__ f2 sin_f32x2(f2 x) { f2 s, c; sincos2<true, false>(x, s, c); return s; }
__device__ __forceinline__ f2 cos_f32x2(f2 x) { f2 s, c; sincos2<false, true>(x, s, c); return c; }
/* two elements of exp_f32 */
__device__ __forceinline__ f2 exp_f32x2(f2 x) {
    const float max_range = +88.3762588501f, min_range = -88.3762588501f;
    f2 t = ffma2(x, 1.4426950408889634073599f, 0.5f);
    f2 n = { floorf(t.x), floorf(t.y) };
    f2 nn = { -n.x, -n.y };
    f2 xr = ffma2(nn, 0.693359375f, x);
    xr = ffma2(nn, -2.12194440e-4f, xr);
    f2 z = poly5(xr, 5.0000001201e-1f, 1.6666665459e-1f, 4.1665795894e-2f,
                     8.3334519073e-3f, 1.3981999507e-3f, 1.9875691500e-4f);
    z = ffma2(z, fmul2(xr, xr), fadd2(xr, mk2(1.f)));
    f2 sc = { fbits((uint32_t) (cvtt_sat(n.x) + 0x7f) << 23), fbits((uint32_t) (cvtt_sat(n.y) + 0x7f) << 23) };
    f2 r = fmul2(z, sc);
    r.x = x.x > max_range ? __int_as_float(0x7f800000) : (x.x < min_range ? 0.f : r.x);
    r.y = x.y > max_range ? __int_as_float(0x7f800000) : (x.y < min_range ? 0.f : r.y);
    return r;
}

/* ---------------- double precision (array_math.h, the `!Single` branches) ---------------- */
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dfma(double a, double b, double c) { return __fma_rn(a, b, c); }
__device__ __forceinline__ double dbits(uint64_t u) { return __longlong_as_double((long long) u); }
__device__ __forceinline__ uint64_t ubits(double d) { return (uint64_t) __double_as_longlong(d); }
/* x86 cvttpd2qq / scalar cvttsd2si semantics */
__device__ __forceinline__ long long cvtt_f64_i64(double x) {
    return (x >= -9223372036854775808.0 && x < 9223372036854775808.0) ? __double2ll_rz(x) : (long long) 0x8000000000000000ull;
}
__device__ __forceinline__ double poly2(double x, double c0, double c1, double c2) {
    double x2 = dmul(x, x);
    return dfma(x2, c2, dfma(x, c1, c0));
}
__device__ __forceinline__ double poly3(double x, double c0, double c1, double c2, double c3) {
    double x2 = dmul(x, x);
    return dfma(x2, dfma(x, c3, c2), dfma(x, c1, c0));
}
__device__ __forceinline__ double poly5(double x, double c0, double c1, double c2, double c3, double c4, double c5) {
    double x2 = dmul(x, x), x4 = dmul(x2, x2);
    return dfma(x2, dfma(x, c3, c2), dfma(x4, dfma(x, c5, c4), dfma(x, c1, c0)));
}

/* array_math.h:261-367 sincos_approx, double branch */
template <bool Sin, bool Cos>
__device__ __forceinline__ void sincos(double x, double &s_out, double &c_out) {
    double xa = fabs(x);
    long long j = cvtt_f64_i64(dmul(xa, 1.2732395447351626862));
    j = (j + 1) & 0xfffffffell;   /* the reference masks with Int(~1u): a 32-bit constant widened to 64 */
    double y = __ll2double_rn(j);
    uint64_t sign_sin = ((uint64_t) j << 61) ^ ubits(x);
    uint64_t sign_cos = (uint64_t) (~(j - 2)) << 61;
    y = dsub(dsub(dsub(xa, dmul(y, 7.85398125648498535156e-1)), dmul(y, 3.77489470793079817668e-8)),
             dmul(y, 2.69515142907905952645e-15));
    double z = dmul(y, y);
    if (xa == dbits(0x7ff0000000000000ull)) z = dbits(~0ull);
    double s = dmul(poly5(z, -1.66666666666666307295e-1, 8.33333333332211858878e-3, -1.98412698295895385996e-4,
                             2.75573136213857245213e-6, -2.50507477628578072866e-8, 1.58962301576546568060e-10), z);
    double c = dmul(poly5(z, 4.16666666666665929218e-2, -1.38888888888730564116e-3, 2.48015872888517045348e-5,
                             -2.75573141792967388112e-7, 2.08757008419747316778e-9, -1.13585365213876817300e-11), z);
    s = dfma(s, y, y);
    c = dfma(c, z, dfma(z, -0.5, 1.0));
    bool polymask = (j & 2) == 0;
    if (Sin) s_out = dbits(ubits(polymask ? s : c) ^ (sign_sin & 0x8000000000000000ull));
    if (Cos) c_out = dbits(ubits(polymask ? c : s) ^ (sign_cos & 0x8000000000000000ull));
}
__device__ __forceinline__ double sin_f64(double x) { double s, c; sincos<true, false>(x, s, c); return s; }
__device__ __forceinline__ double cos_f64(double x) { double s, c; sincos<false, true>(x, s, c); return c; }

/* array_math.h:711-776 exp, double branch */
__device__ __forceinline__ double exp_f64(double x) {
    const double max_range = +7.0943613930310391424428e2, min_range = -7.0943613930310391424428e2;
    bool overflow = x > max_range, underflow = x < min_range;
    double n = floor(dfma(1.4426950408889634073599, x, 0.5));
    double xr = dfma(-n, 6.93145751953125e-1, x);
    xr = dfma(-n, 1.42860682030941723212e-6, xr);
    double z = dmul(xr, xr);
    double p = dmul(poly2(z, 9.99999999999999999910e-1, 3.02994407707441961300e-2, 1.26177193074810590878e-4), xr);
    double q = poly3(z, 2.00000000000000000009e0, 2.27265548208155028766e-1, 2.52448340349684104192e-3, 3.00198505138664455042e-6);
    double pq = __ddiv_rn(p, dsub(q, p));
    z = dadd(dadd(pq, pq), 1.0);
    uint64_t scale = (uint64_t) (cvtt_f64_i64(n) + 0x3ff) << 52;
    double r = dmul(z, dbits(scale));
    return overflow ? dbits(0x7ff0000000000000ull) : (underflow ? 0.0 : r);
}

/* array_math.h:778-898 log, double branch (both sub-branches evaluated and selected, as the IsCuda path does) */
__device__ __forceinline__ double log_f64(double x) {
    bool valid = x >= 0.0;
    uint64_t xi = ubits(x);
    uint64_t exponent_bits = xi & 0x7ff0000000000000ull;
    bool is_normal = (x != 0.0) && (exponent_bits != 0x7ff0000000000000ull);
    long long exponent_i = (long long) (exponent_bits >> 52) - 0x3ff;
    uint64_t mantissa = (xi & ~0x7ff0000000000000ull) | 0x3fe0000000000000ull;
    double xm = dbits(is_normal ? mantissa : xi);
    double e = __ll2double_rn(is_normal ? exponent_i : 0);
    bool e_big = fabs(e) > 2.0;
    bool ge = xm >= 0.70710678118654752440;
    if (ge) e = dadd(e, 1.0);
    /* big exponent: log(x) = z + z^3 P(z)/Q(z), z = 2(x-1)/(x+1) */
    double zb = dsub(xm, 0.5);
    if (ge) zb = dsub(zb, 0.5);
    double yb = dadd(dmul(0.5, ge ? xm : zb), 0.5);
    double x2b = __ddiv_rn(zb, yb);
    double zz = dmul(x2b, x2b);
    zz = dmul(x2b, __ddiv_rn(dmul(zz, poly2(zz, -6.41409952958715622951e1, 1.63866645699558079767e1, -7.89580278884799154124e-1)),
                             poly3(zz, -7.69691943550460008604e2, 3.12093766372244180303e2, -3.56722798256324312549e1, 1.00000000000000000000e0)));
    double r_big = dadd(dfma(-e, 2.121944400546905827679e-4, zz), x2b);
    /* small exponent: log(1+x) = x - x^2/2 + x^3 P(x)/Q(x) */
    double x2s = dsub(ge ? xm : dadd(xm, xm), 1.0);
    double zs = dmul(x2s, x2s);
    double ys = dmul(x2s, __ddiv_rn(dmul(zs, poly5(x2s, 7.70838733755885391666e0, 1.79368678507819816313e1, 1.44989225341610930846e1,
                                                     4.70579119878881725854e0, 4.97494994976747001425e-1, 1.01875663804580931796e-4)),
                                   poly5(x2s, 2.31251620126765340583e1, 7.11544750618563894466e1, 8.29875266912776603211e1,
                                         4.52279145837532221105e1, 1.12873587189167450590e1, 1.00000000000000000000e0)));
    ys = dfma(-e, 2.121944400546905827679e-4, ys);
    double r_small = dadd(x2s, dfma(-0.5, zs, ys));
    double r = e_big ? r_big : r_small;
    r = dfma(e, 0.693359375, r);
    if (x == dbits(0x7ff0000000000000ull)) r = dbits(0x7ff0000000000000ull);
    if (x == 0.0) r = dbits(0xfff0000000000000ull);
    return valid ? r : dbits(~0ull);
}

/* safe_mul / safe_fmadd: src/autodiff/autodiff.cpp:1191-1221 */
__device__ __forceinline__ float mul_nz(float a, float b) {
    return (a == 0.f || b == 0.f) ? 0.f : fmul(a, b);
}
__device__ __forceinline__ float fma_nz(float a, float b, float c) {
    return (a == 0.f || b == 0.f) ? c : ffma(a, b, c);
}
__device__ __forceinline__ double mul_nz(double a, double b) {
    return (a == 0.0 || b == 0.0) ? 0.0 : __dmul_rn(a, b);
}
__device__ __forceinline__ double fma_nz(double a, double b, double c) {
    return (a == 0.0 || b == 0.0) ? c : __fma_rn(a, b, c);
}

/* min/max with the x86 vminps/vmaxps operand rule of the CPU path
   (array_avx.h min_/max_: second operand returned when either is NaN); float: above atan2_f32 */
__device__ __forceinline__ double min_x86(double a, double b) { return a < b ? a : b; }
__device__ __forceinline__ double max_x86(double a, double b) { return a > b ? a : b; }

} // namespace ekm
