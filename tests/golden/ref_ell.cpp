/* The reference's single precision carlson_rf, carlson_rd, carlson_rc, comp_ellint_1 / 2 and ellint_1 / 2
   (include/enoki/special.h) on the AVX2 Packet<float, 8> behind a C ABI, for tests/golden/make_golden_ell.py.  Compiled
   like oracle/_ref: AVX2 + FMA, -ffp-contract=off, and -DNDEBUG (the inputs are in the functions' domains). */
#include <enoki/array.h>
#include <enoki/special.h>
#include <cstddef>

using P8 = enoki::Packet<float, 8>;
using V2 = enoki::Array<P8, 2>;
using V3 = enoki::Array<P8, 3>;

extern "C" {

/* which = 0 carlson_rf(x, y, z), 1 carlson_rd(x, y, z), 2 carlson_rc(x, y); n is a multiple of 8 */
void ref_ell_carlson(int which, const float *x, const float *y, const float *z, float *out, size_t n) {
    for (size_t i = 0; i < n; i += 8) {
        P8 a = enoki::load_unaligned<P8>(x + i), b = enoki::load_unaligned<P8>(y + i), r;
        switch (which) {
            case 0: r = enoki::carlson_rf(V3(a, b, enoki::load_unaligned<P8>(z + i))); break;
            case 1: r = enoki::carlson_rd(V3(a, b, enoki::load_unaligned<P8>(z + i))); break;
            default: r = enoki::carlson_rc(V2(a, b)); break;
        }
        enoki::store_unaligned(out + i, r);
    }
}

/* which = 0 comp_ellint_1(k), 1 comp_ellint_2(k), 2 ellint_1(phi, k), 3 ellint_2(phi, k); n is a multiple of 8 */
void ref_ell_integral(int which, const float *phi, const float *k, float *out, size_t n) {
    for (size_t i = 0; i < n; i += 8) {
        P8 p = enoki::load_unaligned<P8>(phi + i), kk = enoki::load_unaligned<P8>(k + i), r;
        switch (which) {
            case 0: r = enoki::comp_ellint_1(kk); break;
            case 1: r = enoki::comp_ellint_2(kk); break;
            case 2: r = enoki::ellint_1(p, kk); break;
            default: r = enoki::ellint_2(p, kk); break;
        }
        enoki::store_unaligned(out + i, r);
    }
}

}
