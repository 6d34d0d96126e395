/* The reference's single precision sinh, cosh, tanh, asinh, acosh, atanh, cbrt and sincosh (include/enoki/array_math.h,
   AVX2 Packet<float, 8>) behind a C ABI, for tests/golden/make_golden_hyp.py.  Compiled like oracle/_ref: AVX2 + FMA,
   -ffp-contract=off. */
#include <enoki/array.h>
#include <cstddef>

using P8 = enoki::Packet<float, 8>;

extern "C" {

/* which = 0 sinh, 1 cosh, 2 tanh, 3 asinh, 4 acosh, 5 atanh, 6 cbrt, 7 sincosh's sinh, 8 sincosh's cosh; n is a
   multiple of 8 */
void ref_hyp_unary(int which, const float *in, float *out, size_t n) {
    for (size_t i = 0; i < n; i += 8) {
        P8 x = enoki::load_unaligned<P8>(in + i), r;
        switch (which) {
            case 0: r = enoki::sinh(x); break;
            case 1: r = enoki::cosh(x); break;
            case 2: r = enoki::tanh(x); break;
            case 3: r = enoki::asinh(x); break;
            case 4: r = enoki::acosh(x); break;
            case 5: r = enoki::atanh(x); break;
            case 6: r = enoki::cbrt(x); break;
            case 7: r = enoki::sincosh(x).first; break;
            default: r = enoki::sincosh(x).second; break;
        }
        enoki::store_unaligned(out + i, r);
    }
}

}
