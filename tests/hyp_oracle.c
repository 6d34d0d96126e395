/*
 * hyp_oracle.c -- TEST INFRASTRUCTURE: plain-C restatements of the single precision sinh, cosh, tanh, asinh, acosh, atanh
 * and cbrt of the reference's include/enoki/array_math.h, operation for operation as their generic bodies record them on
 * this backend (the evaluator's EK_OP_SINH ... EK_OP_CBRT compute the same sequence on the device, ek_math.cuh).  exp and
 * log are the backend's, restated by oracle/enoki_oracle.c (or_exp / or_log of oracle/liboracle.so, which this file is
 * linked against, so that they are the very code the numpy interpreter calls); rcp, sqrt and division are correctly
 * rounded; value & ~mask and value | mask are the bit operations the backend records.  Where two operands of a recorded
 * operation come in a fixed order (accumulator first), the restatement keeps it, so that NaN payloads follow the same
 * x86 rules as the numpy interpreter running the traced program.
 *
 * Built by tests/hyp_support.py with -ffp-contract=off (every a*b+c stays two roundings unless written fmaf).  The
 * reference CPU path computes rcp with rcpps + one Newton step instead (sinh, cosh and tanh use it), the one place
 * where its results can differ from these.
 *
 *   hy_unary_f32(which, in, out, n): which = 0 sinh, 1 cosh, 2 tanh, 3 asinh, 4 acosh, 5 atanh, 6 cbrt
 */
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <math.h>

#define EXPORT __attribute__((visibility("default")))

float or_exp(float x);
float or_log(float x);

static inline float fbits(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t ubits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
/* x86 cvttps2dq: out-of-range / NaN -> 0x80000000 */
static inline int32_t cvtt(float x) {
    return (x >= -2147483648.f && x < 2147483648.f) ? (int32_t) x : (int32_t) 0x80000000u;
}
/* array_math.h:25-29 */
static inline float poly2(float x, float c0, float c1, float c2) {
    float x2 = x * x;
    return fmaf(x2, c2, fmaf(x, c1, c0));
}

/* array_math.h:31-37 */
static inline float poly3(float x, float c0, float c1, float c2, float c3) {
    float x2 = x * x;
    return fmaf(x2, fmaf(x, c3, c2), fmaf(x, c1, c0));
}
/* array_math.h:39-45 */
static inline float poly4(float x, float c0, float c1, float c2, float c3, float c4) {
    float x2 = x * x, x4 = x2 * x2;
    return fmaf(x2, fmaf(x, c3, c2), fmaf(x, c1, c0) + x4 * c4);
}
/* copysign(r, x) = |r| | (x & sign) (array_router.h:398) */
static inline float copysign_bits(float r, float x) { return fbits((ubits(r) & 0x7fffffffu) | (ubits(x) & 0x80000000u)); }

/* rcp: the correctly rounded quotient */
static inline float rcp(float x) { return 1.f / x; }

/* array_math.h:997-1046 sinh */
static float sinh_f(float x) {
    float x2 = x * x;
    float r_small = fmaf(x2 * x, poly2(x2, (float) 1.66667160211e-1, (float) 8.33028376239e-3, (float) 2.03721912945e-4), x);
    float exp0 = or_exp(x), exp1 = rcp(exp0);
    float r_big = (exp0 - exp1) * 0.5f;
    return fabsf(x) > 1.f ? r_big : r_small;
}
/* array_math.h:1048-1065 cosh */
static float cosh_f(float x) {
    float exp0 = or_exp(x), exp1 = rcp(exp0);
    return (exp1 + exp0) * 0.5f;
}
/* array_math.h:1129-1179 tanh */
static float tanh_f(float x) {
    float x2 = x * x;
    float r_small = poly4(x2, (float) -3.33332819422e-1, (float) 1.33314422036e-1, (float) -5.37397155531e-2,
                              (float) 2.06390887954e-2, (float) -5.70498872745e-3);
    r_small = fmaf(x2 * x, r_small, x);
    float e = or_exp(x + x), e2 = rcp(e + 1.f);
    float r_big = 1.f - (e2 + e2);
    return fabsf(x) >= 0.625f ? r_big : r_small;
}
/* array_math.h:1185-1237 asinh */
static float asinh_f(float x) {
    float x2 = x * x, xa = fabsf(x);
    int big = xa >= (float) 0.51, huge = xa >= (float) 1e10;
    float r_small = poly3(x2, (float) -1.6666288134e-1, (float) 7.4847586088e-2, (float) -4.2699340972e-2,
                              (float) 2.0122003309e-2);
    r_small = fmaf(x2 * x, r_small, x);
    float r_big = or_log((huge ? 0.f : sqrtf(x2 + 1.f)) + xa);                  /* sqrt(x2 + 1) & ~mask_huge */
    if (huge) r_big = r_big + (float) M_LN2;                                     /* r_big[mask_huge] += M_LN2 */
    r_big = copysign_bits(r_big, x);
    return big ? r_big : r_small;
}
/* array_math.h:1239-1293 acosh */
static float acosh_f(float x) {
    float x1 = x - 1.f;
    int big = x1 >= (float) 0.49, huge = x1 >= (float) 1e10;
    float r_small = poly4(x1, (float) 1.4142135263e+0, (float) -1.1784741703e-1, (float) 2.6454905019e-2,
                              (float) -7.5272886713e-3, (float) 1.7596881071e-3);
    r_small = sqrtf(x1) * r_small;
    if (x1 < 0.f) r_small = fbits(0xffffffffu);                                  /* r_small |= x1 < 0 */
    float r_big = or_log((huge ? 0.f : sqrtf(fmaf(x, x, -1.f))) + x);          /* fmsub(x, x, 1) */
    if (huge) r_big = r_big + (float) M_LN2;
    return big ? r_big : r_small;
}
/* array_math.h:1295-1348 atanh */
static float atanh_f(float x) {
    float xa = fabsf(x), x2 = x * x;
    float r_small = poly4(x2, (float) 3.33337300303e-1, (float) 1.99782164500e-1, (float) 1.46691431730e-1,
                              (float) 8.24370301058e-2, (float) 1.81740078349e-1);
    r_small = fmaf(x2 * x, r_small, x);
    float r_big = or_log((xa + 1.f) / (1.f - xa)) * 0.5f;
    r_big = copysign_bits(r_big, x);
    return xa >= 0.5f ? r_big : r_small;
}
/* array_math.h:900-954 cbrt, with frexp :682-709 and ldexp :677-680 */
static float cbrt_f(float x) {
    const float CBRT2 = (float) 1.25992104989487316477, CBRT4 = (float) 1.58740105196819947475,
                THIRD = (float) (1.0 / 3.0);
    float xa = fabsf(x);
    uint32_t xi = ubits(xa), exponent_bits = xi & 0x7f800000u;
    int is_normal = exponent_bits != 0x7f800000u && xa != 0.f;
    float xm = fbits(is_normal ? (xi & 0x807fffffu) | 0x3f000000u : xi);
    float xe = (float) (is_normal ? (int32_t) (exponent_bits >> 23) - 0x7f : 0) + 1.f;
    float xea = fabsf(xe), xea1 = floorf(xea * THIRD);
    float rem = fmaf(xea1, -3.f, xea);                                           /* fnmadd(xea1, 3, xea) */
    xm = poly4(xm, (float) 0.40238979564544752126924, (float) 1.1399983354717293273738,
                   (float) -0.95438224771509446525043, (float) 0.54664601366395524503440,
                   (float) -0.13466110473359520655053);
    float f1 = xe >= 0.f ? CBRT2 : 1.f / CBRT2, f2 = xe >= 0.f ? CBRT4 : 1.f / CBRT4;
    float f = rem == 1.f ? f1 : f2;
    if (rem != 0.f) xm = f * xm;                                                 /* xm[neq(rem, 0)] *= f */
    float e = fbits(ubits(xea1) ^ (ubits(xe) & 0x80000000u));                    /* mulsign(xea1, xe) */
    float r = fbits(((uint32_t) cvtt(e) + 0x7fu) << 23) * xm;                    /* ldexp(xm, e) */
    r = fbits(ubits(r) ^ (ubits(x) & 0x80000000u));                             /* mulsign(r, x) */
    r = r - (r - x / (r * r)) * THIRD;
    return fabsf(x) < INFINITY ? r : x;
}

static float hy_one(int which, float x) {
    switch (which) {
        case 0: return sinh_f(x);
        case 1: return cosh_f(x);
        case 2: return tanh_f(x);
        case 3: return asinh_f(x);
        case 4: return acosh_f(x);
        case 5: return atanh_f(x);
        default: return cbrt_f(x);
    }
}

EXPORT void hy_unary_f32(int which, const float *in, float *out, size_t n) {
    for (size_t i = 0; i < n; ++i) out[i] = hy_one(which, in[i]);
}
