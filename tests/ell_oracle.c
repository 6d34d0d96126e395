/*
 * ell_oracle.c -- TEST INFRASTRUCTURE: plain-C restatements of the single precision Carlson integrals carlson_rf,
 * carlson_rd and carlson_rc of the reference's include/enoki/special.h, operation for operation as their generic bodies
 * record them on this backend (the evaluator's EK_OP_CARLSON_RF ... EK_OP_CARLSON_RC compute the same sequence on the
 * device, ek_math.cuh).  sqrt, rcp and division are correctly rounded, hmax follows the x86 operand rule (the second
 * operand when the comparison is false), fnmadd / fmadd are single fmaf calls, and the duplication loop runs one element
 * at a time: evaluate the loop head, stop when !(eps > threshold) or after the tenth head, else update.
 *
 * Built by tests/ell_support.py with -ffp-contract=off (every a*b+c stays two roundings unless written fmaf).
 *
 *   el_ternary_f32(which, x, y, z, out, n): which = 0 carlson_rf, 1 carlson_rd
 *   el_binary_f32(x, y, out, n):            carlson_rc
 */
#include <stddef.h>
#include <math.h>

#define EXPORT __attribute__((visibility("default")))

static inline float max_x86(float a, float b) { return a > b ? a : b; }

/* special.h:325-366 */
static float carlson_rf(float x, float y, float z) {
    const float thr = (float) 0.070154;
    float X, Y, Z, mu_inv;
    for (int it = 1;; ++it) {
        float sx = sqrtf(x), sy = sqrtf(y), sz = sqrtf(z);
        float lambda = fmaf(sx, sz, fmaf(sz, sy, sy * sx));
        float mu = ((x + y) + z) * (float) (1.0 / 3.0);
        mu_inv = 1.f / mu;
        X = fmaf(-x, mu_inv, 1.f); Y = fmaf(-y, mu_inv, 1.f); Z = fmaf(-z, mu_inv, 1.f);
        float eps = max_x86(max_x86(fabsf(X), fabsf(Y)), fabsf(Z));
        if (!(eps > thr) || it == 10) break;
        x = (x + lambda) * 0.25f; y = (y + lambda) * 0.25f; z = (z + lambda) * 0.25f;
    }
    float e2 = X * Y - Z * Z, e3 = (X * Y) * Z;
    float er = (((float) (1.0 / 24.0) * e2 - (float) (1.0 / 10.0)) - (float) (3.0 / 44.0) * e3) * e2 +
               (float) (1.0 / 14.0) * e3;
    return sqrtf(mu_inv) * (1.f + er);
}

/* special.h:379-432 */
static float carlson_rd(float x, float y, float z) {
    const float thr = (float) (0.070154 * 0.6), w0 = (float) (1.0 / 5.0), w2 = (float) (3.0 / 5.0);
    float X, Y, Z, mu_inv, sum = 0.f, num = 1.f;
    for (int it = 1;; ++it) {
        float sx = sqrtf(x), sy = sqrtf(y), sz = sqrtf(z);
        float lambda = fmaf(sx, sz, fmaf(sz, sy, sy * sx));
        float mu = (x * w0 + y * w0) + z * w2;
        mu_inv = 1.f / mu;
        X = fmaf(-x, mu_inv, 1.f); Y = fmaf(-y, mu_inv, 1.f); Z = fmaf(-z, mu_inv, 1.f);
        float eps = max_x86(max_x86(fabsf(X), fabsf(Y)), fabsf(Z));
        if (!(eps > thr) || it == 10) break;
        sum = sum + num / (sz * (z + lambda));
        num = num * 0.25f;
        x = (x + lambda) * 0.25f; y = (y + lambda) * 0.25f; z = (z + lambda) * 0.25f;
    }
    float ea = X * Y, eb = Z * Z, ec = ea - eb, ed = fmaf(-6.f, eb, ea), ee = fmaf(ec, 2.f, ed);
    float p = ed * ((-(float) (3.0 / 14.0) + (float) (9.0 / 88.0) * ed) - (0.25f * Z) * ee) +
              Z * ((float) (1.0 / 6.0) * ee + Z * (-(float) (9.0 / 22.0) * ec + (Z * (float) (3.0 / 26.0)) * ea));
    return 3.f * sum + ((num * mu_inv) * sqrtf(mu_inv)) * (1.f + p);
}

/* special.h:445-482 */
static float carlson_rc(float x, float y) {
    const float thr = (float) (0.070154 * 0.48);
    float inv_mu, s;
    for (int it = 1;; ++it) {
        float lambda = sqrtf(x) * sqrtf(y);
        lambda = lambda + (lambda + y);
        float mu = fmaf(x, (float) (1.0 / 3.0), y * (float) (2.0 / 3.0));
        inv_mu = 1.f / mu;
        s = (y - mu) * inv_mu;
        if (!(fabsf(s) > thr) || it == 10) break;
        x = (x + lambda) * 0.25f; y = (y + lambda) * 0.25f;
    }
    return sqrtf(inv_mu) * (1.f + (s * s) * (0.3f + s * ((float) (1.0 / 7.0) + s * (0.375f + s * (float) (9.0 / 22.0)))));
}

EXPORT void el_ternary_f32(int which, const float *x, const float *y, const float *z, float *out, size_t n) {
    for (size_t i = 0; i < n; ++i) out[i] = which == 0 ? carlson_rf(x[i], y[i], z[i]) : carlson_rd(x[i], y[i], z[i]);
}

EXPORT void el_binary_f32(const float *x, const float *y, float *out, size_t n) {
    for (size_t i = 0; i < n; ++i) out[i] = carlson_rc(x[i], y[i]);
}
