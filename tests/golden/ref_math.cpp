/* The reference's single precision pow, frexp, hypot (include/enoki/array_math.h), dawson and erfi
   (include/enoki/special.h) on the AVX2 Packet<float, 8> behind a C ABI, for tests/golden/make_golden_math.py.  Compiled
   like oracle/_ref: AVX2 + FMA, -ffp-contract=off. */
#include <enoki/array.h>
#include <enoki/special.h>
#include <cstddef>

using P8 = enoki::Packet<float, 8>;

extern "C" {

/* which = 0 pow, 1 hypot; n is a multiple of 8 */
void ref_math_binary(int which, const float *x, const float *y, float *out, size_t n) {
    for (size_t i = 0; i < n; i += 8) {
        P8 a = enoki::load_unaligned<P8>(x + i), b = enoki::load_unaligned<P8>(y + i), r;
        switch (which) {
            case 0: r = enoki::pow(a, b); break;
            default: r = enoki::hypot(a, b); break;
        }
        enoki::store_unaligned(out + i, r);
    }
}

/* which = 0 frexp mantissa, 1 frexp exponent, 2 dawson, 3 erfi; n is a multiple of 8 */
void ref_math_unary(int which, const float *x, float *out, size_t n) {
    for (size_t i = 0; i < n; i += 8) {
        P8 a = enoki::load_unaligned<P8>(x + i), r;
        switch (which) {
            case 0: r = enoki::frexp(a).first; break;
            case 1: r = enoki::frexp(a).second; break;
            case 2: r = enoki::dawson(a); break;
            default: r = enoki::erfi(a); break;
        }
        enoki::store_unaligned(out + i, r);
    }
}

}
