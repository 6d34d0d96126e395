/*
 * math_oracle.c -- TEST INFRASTRUCTURE: plain-C restatements of the single precision pow, frexp and hypot of
 * the reference's include/enoki/array_math.h and dawson and erfi of include/enoki/special.h, operation for operation as
 * their generic bodies record them on this backend (the evaluator's EK_OP_POW ... EK_OP_ERFI compute the same sequence
 * on the device, ek_math.cuh).  exp and log are the backend's, restated by oracle/enoki_oracle.c (or_exp / or_log of
 * oracle/liboracle.so, which this file is linked against); division and sqrt are correctly rounded, min / max follow the
 * x86 operand rule (the second operand when the comparison is false).  Each operation keeps the
 * operand order of the recorded program (accumulator first), so that NaN payloads follow the same x86 rules as the numpy
 * interpreter running the traced program.
 *
 * Built by tests/math_support.py with -ffp-contract=off (every a*b+c stays two roundings unless written fmaf).
 *
 *   mt_binary_f32(which, x, y, out, n): which = 0 pow, 1 hypot
 *   mt_unary_f32(which, x, out, n):     which = 0 frexp mantissa, 1 frexp exponent, 2 dawson, 3 erfi
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

/* array_math.h:56-63 poly6 */
static inline float poly6(float x, float c0, float c1, float c2, float c3, float c4, float c5, float c6) {
    float x2 = x * x, x4 = x2 * x2;
    return fmaf(x4, fmaf(x2, c6, fmaf(x, c5, c4)), fmaf(x2, fmaf(x, c3, c2), fmaf(x, c1, c0)));
}
/* array_math.h:65-72 poly7 */
static inline float poly7(float x, float c0, float c1, float c2, float c3, float c4, float c5, float c6, float c7) {
    float x2 = x * x, x4 = x2 * x2;
    return fmaf(x4, fmaf(x2, fmaf(x, c7, c6), fmaf(x, c5, c4)), fmaf(x2, fmaf(x, c3, c2), fmaf(x, c1, c0)));
}

/* array_math.h:956-958 */
static float pow_f(float x, float y) { return or_exp(or_log(x) * y); }
/* array_math.h:682-709 */
static int frexp_normal(float x) { return x != 0.f && (ubits(x) & 0x7f800000u) != 0x7f800000u; }
static float frexp_m(float x) { return frexp_normal(x) ? fbits((ubits(x) & ~0x7f800000u) | 0x3f000000u) : x; }
static float frexp_e(float x) {
    return (float) (frexp_normal(x) ? (int32_t) ((ubits(x) & 0x7f800000u) >> 23) - 0x7f : 0);
}
/* array_math.h:1362-1379 */
static float hypot_f(float a, float b) {
    float abs_a = fabsf(a), abs_b = fabsf(b);
    float maxval = abs_a > abs_b ? abs_a : abs_b, minval = abs_a < abs_b ? abs_a : abs_b, ratio = minval / maxval;
    float big = maxval * sqrtf(1.f + ratio * ratio), sum = abs_a + abs_b;
    return (abs_a < INFINITY && abs_b < INFINITY && ratio < INFINITY) ? big : sum;
}
/* special.h:249-265 */
static float dawson_f(float x) {
    float x2 = x * x;
    float num = poly6(x2, (float) 1.00000080272429, (float) 9.18170212243285e-2, (float) 4.25835373536124e-2,
                          (float) 6.0536496345054e-3, (float) 9.88555033724111e-4, (float) 3.64943550840577e-5,
                          (float) 1.55942290996993e-5);
    float denom = poly7(x2, 1.f, (float) 7.58517175815194e-1, (float) 2.81364355593059e-1, (float) 6.81783097841267e-2,
                            (float) 1.13586116798019e-2, (float) 1.92020805811771e-3, (float) 5.74217664074868e-5,
                            (float) 3.11884331363595e-5);
    return num / denom * x;
}
/* special.h:267-271 */
static float erfi_f(float x) { return (float) M_2_SQRTPI * dawson_f(x) * or_exp(x * x); }

EXPORT void mt_binary_f32(int which, const float *x, const float *y, float *out, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        switch (which) {
            case 0: out[i] = pow_f(x[i], y[i]); break;
            default: out[i] = hypot_f(x[i], y[i]); break;
        }
    }
}

EXPORT void mt_unary_f32(int which, const float *x, float *out, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        switch (which) {
            case 0: out[i] = frexp_m(x[i]); break;
            case 1: out[i] = frexp_e(x[i]); break;
            case 2: out[i] = dawson_f(x[i]); break;
            default: out[i] = erfi_f(x[i]); break;
        }
    }
}
