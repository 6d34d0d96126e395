/* The reference's single precision erf, erfc, erfinv, lgamma and tgamma (include/enoki/special.h, AVX2 Packet<float, 8>)
   behind a C ABI, for tests/golden/make_golden_special.py.  Compiled like oracle/_ref: AVX2 + FMA, -ffp-contract=off. */
#include <enoki/array.h>
#include <enoki/special.h>
#include <cstddef>

using P8 = enoki::Packet<float, 8>;

extern "C" {

/* which = 0 erf, 1 erfc, 2 erfinv, 3 lgamma, 4 tgamma; n is a multiple of 8 */
void ref_special_unary(int which, const float *in, float *out, size_t n) {
    for (size_t i = 0; i < n; i += 8) {
        P8 x = enoki::load_unaligned<P8>(in + i), r;
        switch (which) {
            case 0: r = enoki::erf(x); break;
            case 1: r = enoki::erfc(x); break;
            case 2: r = enoki::erfinv(x); break;
            case 3: r = enoki::lgamma(x); break;
            default: r = enoki::tgamma(x); break;
        }
        enoki::store_unaligned(out + i, r);
    }
}

}
