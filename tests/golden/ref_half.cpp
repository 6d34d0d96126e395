/* The reference's scalar half (include/enoki/half.h, compiled with -mf16c: F16C's vcvtps2ph / vcvtph2ps) behind a C ABI,
   for tests/golden/make_golden_f16.py.  Type codes are the ek_type values of include/enoki_b200.h. */
#include <immintrin.h>              /* (half.h uses the F16C intrinsics without including their header) */
#include <enoki/half.h>
#include <cstddef>
#include <cstdint>
#include <cstring>

using enoki::half;

template <typename S> static void from(const void *in, uint16_t *out, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        half h(((const S *) in)[i]);            /* half(Value v) = float32_to_float16(float(v)) */
        memcpy(out + i, &h, 2);
    }
}

extern "C" {

int ref_half_from(int src, const void *in, uint16_t *out, size_t n) {
    switch (src) {
        case 1:  from<int8_t>(in, out, n); return 0;
        case 2:  from<uint8_t>(in, out, n); return 0;
        case 3:  from<int16_t>(in, out, n); return 0;
        case 4:  from<uint16_t>(in, out, n); return 0;
        case 5:  from<int32_t>(in, out, n); return 0;
        case 6:  from<uint32_t>(in, out, n); return 0;
        case 7:  from<int64_t>(in, out, n); return 0;
        case 8:  from<uint64_t>(in, out, n); return 0;
        case 10: from<float>(in, out, n); return 0;
        case 11: from<double>(in, out, n); return 0;
        default: return -1;
    }
}

void ref_half_to_float(const uint16_t *in, float *out, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        half h;
        memcpy(&h, in + i, 2);
        out[i] = (float) h;
    }
}

}
