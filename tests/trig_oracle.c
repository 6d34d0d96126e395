/*
 * trig_oracle.c -- TEST INFRASTRUCTURE: plain-C restatements of the single precision tan, cot, asin, acos, atan and
 * atan2 of the reference's include/enoki/array_math.h, operation for operation as their generic bodies record them on
 * this backend (the evaluator's EK_OP_TAN ... EK_OP_ATAN2 compute the same sequence on the device, ek_math.cuh).
 *
 * Built by tests/trig_support.py with -ffp-contract=off (every a*b+c stays two roundings unless written fmaf).  rcp and
 * 1 / x are the correctly rounded quotient the backend uses (DESIGN.md §4); the reference CPU path computes tan / cot's
 * rcp with rcpps + one Newton step instead, and its min / max pick the other operand of a NaN pair (atan2 with one NaN
 * operand): the two places where its results can differ from these.
 *
 *   tr_unary_f32(which, in, out, n): which = 0 tan, 1 cot, 2 asin, 3 acos, 4 atan
 *   tr_atan2_f32(y, x, out, n):       atan2(y, x)
 *   tr_tancot_f32_rcp(tan, in, out, branch, recip_kind, n): tan (tan = 1) or cot with the reciprocal computed as the
 *       correctly rounded float quotient (recip_kind 0) or the double quotient rounded to float (1); branch[i] = 1 where
 *       the element took the reciprocal branch
 */
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <math.h>

static inline float fbits(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t ubits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

/* x86 cvttps2dq: out-of-range / NaN -> 0x80000000 */
static inline int32_t cvtt(float x) {
    return (x >= -2147483648.f && x < 2147483648.f) ? (int32_t) x : (int32_t) 0x80000000u;
}
/* the evaluator's min / max (ek_math.cuh min_x86 / max_x86): the second operand when either is NaN */
static inline float min_x86(float a, float b) { return a < b ? a : b; }
static inline float max_x86(float a, float b) { return a > b ? a : b; }

/* array_math.h:39-45 */
static inline float poly4(float x, float c0, float c1, float c2, float c3, float c4) {
    float x2 = x * x, x4 = x2 * x2;
    return fmaf(x2, fmaf(x, c3, c2), fmaf(x, c1, c0) + c4 * x4);
}
/* array_math.h:47-54 */
static inline float poly5(float x, float c0, float c1, float c2, float c3, float c4, float c5) {
    float x2 = x * x, x4 = x2 * x2;
    return fmaf(x2, fmaf(x, c3, c2), fmaf(x4, fmaf(x, c5, c4), fmaf(x, c1, c0)));
}
/* array_math.h:56-63 */
static inline float poly6(float x, float c0, float c1, float c2, float c3, float c4, float c5, float c6) {
    float x2 = x * x, x4 = x2 * x2;
    return fmaf(x4, fmaf(x2, c6, fmaf(x, c5, c4)), fmaf(x2, fmaf(x, c3, c2), fmaf(x, c1, c0)));
}

/* array_math.h:369-442 tancot_approx<Tan>, single precision branch; *branch = 1 where the reciprocal is taken */
static float tancot(int tan, float x, int recip_kind, int *branch) {
    float xa = fabsf(x);
    int32_t j = cvtt(xa * (float) 1.2732395447351626862);
    j = (int32_t) (((uint32_t) j + 1u) & ~1u);
    float y = (float) j;
    y = xa - y * (float) 0.78515625 - y * (float) 2.4187564849853515625e-4 - y * (float) 3.77489497744594108e-8;
    float z = y * y;
    if (xa == INFINITY) z = fbits(0xffffffffu);                          /* z |= eq(xa, inf) */
    float r = poly5(z, (float) 3.33331568548e-1, (float) 1.33387994085e-1, (float) 5.34112807005e-2,
                       (float) 2.44301354525e-2, (float) 3.11992232697e-3, (float) 9.38540185543e-3);
    r = fmaf(r, z * y, y);
    if (xa < (float) 1e-4) r = y;                                        /* r[xa < 1e-4] = y */
    int recip = tan ? (j & 2) != 0 : (j & 2) == 0;
    if (branch) *branch = recip;
    if (recip) r = recip_kind ? (float) (1.0 / (double) r) : 1.f / r;    /* r[recip_mask] = rcp(r) */
    uint32_t sign = ((uint32_t) j << 30) ^ ubits(x);
    return fbits(ubits(r) ^ (sign & 0x80000000u));                       /* mulsign(r, sign) */
}

/* array_math.h:489-507 / :571-585: z1 of asin / acos, *big = |x| > 0.5 */
static inline float asincos_core(float x, float c0, int *big) {
    float xa = fabsf(x), x2 = x * x;
    *big = xa > 0.5f;
    float x1 = 0.5f * (1.f - xa);
    float x3 = *big ? x1 : x2;
    float x4 = *big ? sqrtf(x1) : xa;
    float z1 = poly4(x3, c0, 7.4953002686e-2f, 4.5470025998e-2f, 2.4181311049e-2f, 4.2163199048e-2f);
    return fmaf(z1, x3 * x4, x4);
}
static inline float copysign_bits(float a, float b) { return fbits((ubits(a) & 0x7fffffffu) | (ubits(b) & 0x80000000u)); }

/* array_math.h:474-553 */
static float asin_f(float x) {
    int big;
    float z1 = asincos_core(x, 1.6666752422e-1f, &big);
    float r = big ? (float) M_PI_2 - (z1 + z1) : z1;
    return copysign_bits(r, x);
}
/* array_math.h:555-590 */
static float acos_f(float x) {
    int big;
    float z1 = asincos_core(x, 1.666675242e-1f, &big);
    float z2 = z1 + z1;
    if (x < 0.f) z2 = (float) M_PI - z2;
    float z3 = (float) M_PI_2 - copysign_bits(z1, x);
    return big ? z2 : z3;
}
/* array_math.h:603-664: atan2(y, x) */
static float atan2_f(float y, float x) {
    float abs_x = fabsf(x), abs_y = fabsf(y);
    float min_val = min_x86(abs_y, abs_x), max_val = max_x86(abs_x, abs_y);
    float scale = 1.f / max_val, scaled_min = min_val * scale, z = scaled_min * scaled_min;
    float t = poly6(z, (float) 0.99999934166683966009, (float) -0.33326497518773606976, (float) +0.19881342388439013552,
                       (float) -0.13486708938456973185, (float) +0.083863120428809689910, (float) -0.037006525670417265220,
                       (float) 0.0078613793713198150252);
    t = t * scaled_min;
    if (abs_y > abs_x) t = (float) M_PI_2 - t;
    if (x < 0.f) t = (float) M_PI - t;
    float r = y < 0.f ? fbits(ubits(t) ^ 0x80000000u) : t;
    return max_val != 0.f ? r : 0.f;                                      /* r &= neq(max_val, 0) */
}

void tr_unary_f32(int which, const float *in, float *out, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        float x = in[i], r;
        switch (which) {
            case 0: r = tancot(1, x, 0, NULL); break;
            case 1: r = tancot(0, x, 0, NULL); break;
            case 2: r = asin_f(x); break;
            case 3: r = acos_f(x); break;
            default: r = atan2_f(x, 1.f); break;                         /* array_math.h:666-668 */
        }
        out[i] = r;
    }
}

void tr_atan2_f32(const float *y, const float *x, float *out, size_t n) {
    for (size_t i = 0; i < n; ++i) out[i] = atan2_f(y[i], x[i]);
}

void tr_tancot_f32_rcp(int tan, const float *in, float *out, int32_t *branch, int recip_kind, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        int b;
        out[i] = tancot(tan, in[i], recip_kind, &b);
        branch[i] = b;
    }
}
