/* The reference's single precision cot and atan2 (include/enoki/array_math.h, AVX2 Packet<float, 8>) behind a C ABI, for
   tests/golden/make_golden_trig.py.  Compiled like oracle/_ref: AVX2 + FMA, -ffp-contract=off. */
#include <enoki/array.h>
#include <cstddef>
#include <cstring>

using P8 = enoki::Packet<float, 8>;

extern "C" {

/* which = 0 tan, 1 cot, 2 asin, 3 acos, 4 atan; n is a multiple of 8 */
void ref_trig_unary(int which, const float *in, float *out, size_t n) {
    for (size_t i = 0; i < n; i += 8) {
        P8 x = enoki::load_unaligned<P8>(in + i), r;
        switch (which) {
            case 0: r = enoki::tan(x); break;
            case 1: r = enoki::cot(x); break;
            case 2: r = enoki::asin(x); break;
            case 3: r = enoki::acos(x); break;
            default: r = enoki::atan(x); break;
        }
        enoki::store_unaligned(out + i, r);
    }
}

/* atan2(y, x); n is a multiple of 8 */
void ref_trig_atan2(const float *y, const float *x, float *out, size_t n) {
    for (size_t i = 0; i < n; i += 8)
        enoki::store_unaligned(out + i, enoki::atan2(enoki::load_unaligned<P8>(y + i), enoki::load_unaligned<P8>(x + i)));
}

}
