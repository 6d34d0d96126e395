/*
 * special_oracle.c -- TEST INFRASTRUCTURE: plain-C restatements of the single precision erf, erfc, erfinv, lgamma and
 * tgamma of the reference's include/enoki/special.h, operation for operation as their generic bodies record them on this
 * backend (the evaluator's EK_OP_ERF ... EK_OP_TGAMMA compute the same sequence on the device, ek_math.cuh).  exp, log
 * and sin are the backend's, restated by oracle/enoki_oracle.c (or_exp / or_log / or_sin of oracle/liboracle.so, which
 * this file is linked against, so that they are the very code the numpy interpreter calls); rcp and division are
 * correctly rounded, round is rintf (nearest even), negation is a sign flip.  Each operation keeps the operand order of
 * the recorded program (accumulator first), so that NaN payloads follow the same x86 rules as the numpy interpreter
 * running the traced program; the polynomials are evaluated in the order the program records them.
 *
 * Built by tests/special_support.py with -ffp-contract=off (every a*b+c stays two roundings unless written fmaf).  The
 * reference CPU path computes rcp with rcpps + one Newton step instead (erf and erfc take it for |x| >= 1), the one
 * place where its results can differ from these.
 *
 *   sp_unary_f32(which, in, out, n): which = 0 erf, 1 erfc, 2 erfinv, 3 lgamma, 4 tgamma
 */
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <math.h>

#define EXPORT __attribute__((visibility("default")))

float or_exp(float x);
float or_log(float x);
float or_sin(float x);

static inline float fbits(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t ubits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float neg(float x) { return fbits(ubits(x) ^ 0x80000000u); }

/* array_math.h:56-63 poly6 */
static inline float poly6(float x, float c0, float c1, float c2, float c3, float c4, float c5, float c6) {
    float m = fmaf(x, c3, c2), lo = fmaf(x, c1, c0), x2 = x * x;
    lo = fmaf(x2, m, lo);
    float hi = fmaf(x2, c6, fmaf(x, c5, c4));
    return fmaf(x2 * x2, hi, lo);
}
/* array_math.h:65-72 poly7 */
static inline float poly7(float x, float c0, float c1, float c2, float c3, float c4, float c5, float c6, float c7) {
    float x2 = x * x;
    float hi = fmaf(x2, fmaf(x, c7, c6), fmaf(x, c5, c4));
    float lo = fmaf(x2, fmaf(x, c3, c2), fmaf(x, c1, c0));
    return fmaf(x2 * x2, hi, lo);
}
/* array_math.h:74-82 poly8 */
static inline float poly8(float x, float c0, float c1, float c2, float c3, float c4, float c5, float c6, float c7,
                          float c8) {
    float x2 = x * x, x4 = x2 * x2, x8 = x4 * x4;
    float lo = fmaf(x, c1, c0) + x8 * c8;
    lo = fmaf(fmaf(x, c3, c2), x2, lo);
    float hi = fmaf(x2, fmaf(x, c7, c6), fmaf(x, c5, c4));
    return fmaf(hi, x4, lo);
}

/* special.h:56-129 erfc<T, false>, single precision branch */
static float erfc_core(float x) {
    float xa = fabsf(x), q = 1.f / xa, y = q * q;
    float p_small = poly8(y, (float) 5.638259427386472e-1, (float) -2.741127028184656e-1, (float) 3.404879937665872e-1,
                             (float) -4.944515323274145e-1, (float) 6.210004621745983e-1, (float) -5.824733027278666e-1,
                             (float) 3.687424674597105e-1, (float) -1.387039388740657e-1, (float) 2.326819970068386e-2);
    float p_large = poly7(y, (float) 5.641895067754075e-1, (float) -2.820767439740514e-1, (float) 4.218463358204948e-1,
                             (float) -1.015265279202700e+0, (float) 2.921019019210786e+0, (float) -7.495518717768503e+0,
                             (float) 1.297719955372516e+1, (float) -1.047766399936249e+1);
    float sel = xa > 2.f ? p_large : p_small;
    float r = (or_exp(neg(x) * x) * q) * sel;
    return x < 0.f ? 2.f - r : r;
}
/* special.h:131-164 erf<T, false>, single precision branch */
static float erf_core(float x) {
    return poly6(x * x, (float) 1.128379165726710e+0, (float) -3.761262582423300e-1, (float) 1.128358514861418e-1,
                        (float) -2.685381193529856e-2, (float) 5.188327685732524e-3, (float) -8.010193625184903e-4,
                        (float) 7.853861353153693e-5) * x;
}
static float erf_f(float x) { float c = 1.f - erfc_core(x), e = erf_core(x); return fabsf(x) > 1.f ? c : e; }
static float erfc_f(float x) { float c = erfc_core(x), e = 1.f - erf_core(x); return fabsf(x) < 1.f ? e : c; }

/* special.h:222-246 erfinv */
static float erfinv_f(float x) {
    float s = 1.f - x;
    float w = neg(or_log((1.f + x) * s));
    float p2 = poly8(sqrtf(w) - 3.f, (float) 2.83297682, (float) 1.00167406, (float) 0.00943887047,
                     (float) -0.0076224613, (float) 0.00573950773, (float) -0.00367342844, (float) 0.00134934322,
                     (float) 0.000100950558, (float) -0.000200214257);
    float p1 = poly8(w - 2.5f, (float) 1.50140941, (float) 0.246640727, (float) -0.00417768164, (float) -0.00125372503,
                     (float) 0.00021858087, (float) -4.39150654e-06, (float) -3.5233877e-06, (float) 3.43273939e-07,
                     (float) 2.81022636e-08);
    return (w < 5.f ? p1 : p2) * x;
}

/* special.h:275-309 lgamma: the sum starts from a recorded literal 0 */
static float lgamma_f(float x_) {
    const float pi = (float) 3.14159265358979323846;
    int reflect = x_ < 0.5f;
    float x = reflect ? neg(x_) : x_ - 1.f;
    float sum = (float) -0.5395239384953e-5 / (x + 6.f) + 0.f;
    sum = (float) 0.1208650973866179e-2 / (x + 5.f) + sum;
    sum = (float) -1.231739572450155 / (x + 4.f) + sum;
    sum = (float) 24.01409824083091 / (x + 3.f) + sum;
    sum = (float) -86.50532032941677 / (x + 2.f) + sum;
    sum = (float) 76.18009172947146 / (x + 1.f) + sum;
    sum = sum + (float) 1.000000000190015;
    float t = or_log(sum) + (float) 0.91893853320467274178;
    float b = (x + 5.f) + 0.5f;
    t = t - b;
    float result = (x + 0.5f) * or_log(b) + t;
    float refl = or_log(fabsf(pi / or_sin(pi * x_))) - result;
    if (reflect) result = refl;
    if (rintf(x_) == x_ && reflect) result = INFINITY;
    return result;
}

static float sp_one(int which, float x) {
    switch (which) {
        case 0: return erf_f(x);
        case 1: return erfc_f(x);
        case 2: return erfinv_f(x);
        case 3: return lgamma_f(x);
        default: return or_exp(lgamma_f(x));
    }
}

EXPORT void sp_unary_f32(int which, const float *in, float *out, size_t n) {
    for (size_t i = 0; i < n; ++i) out[i] = sp_one(which, in[i]);
}
