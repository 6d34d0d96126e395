/* Float16 storage through include/enoki/cuda.h (CUDAArray<half>): an image of half values is loaded, widened to float,
   filtered with gathers of its neighbours, rounded back to half and scattered into a mirrored image -- "load half,
   compute in float, store half".  The same computation on the host with the reference's enoki::half (half.h: the
   F16C conversions) gives the expected bits.  Also: a half literal, the bit casts to and from uint16_t.
   Prints "half_check ok" and exits 0 when every bit matches.  Written from scratch. */
#include <enoki/cuda.h>
#include <enoki/half.h>
#include <cstdio>
#include <cstring>
#include <vector>

using namespace enoki;
using FloatC = CUDAArray<float>;
using HalfC = CUDAArray<half>;
using UInt16C = CUDAArray<uint16_t>;
using UInt32C = CUDAArray<uint32_t>;
using MaskC = mask_t<UInt32C>;

static std::vector<uint16_t> bits_of(const HalfC &a) {
    std::vector<uint16_t> v(a.size());
    a.eval();
    cuda_memcpy_from_device(v.data(), a.data(), v.size() * 2);
    return v;
}

int main() {
    const uint32_t W = 1021, H = 769, n = W * H;
    std::vector<half> img(n);
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t h = i * 2654435761u;
        h ^= h >> 15;
        img[i] = half((float) (h & 0xffffu) * (6.f / 65535.f) - 3.f);
    }

    HalfC d = HalfC::copy(img.data(), n);
    UInt32C idx = arange<UInt32C>(n), x = idx % W;
    UInt32C left = select(x > 0u, idx - 1u, idx), right = select(x < W - 1, idx + 1u, idx);
    FloatC c = FloatC(d), l = FloatC(gather<HalfC>(d, left)), r = FloatC(gather<HalfC>(d, right));
    FloatC blur = (l + c * 2.f + r) * 0.25f;
    FloatC y = blur * blur * 0.5f - 0.125f;
    HalfC out = HalfC(y);
    HalfC mirrored = zero<HalfC>(n);
    scatter(mirrored, out, UInt32C(n - 1) - idx, MaskC(true));

    std::vector<uint16_t> want(n), want_m(n);
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t xi = i % W, li = xi > 0 ? i - 1 : i, ri = xi < W - 1 ? i + 1 : i;
        float cf = (float) img[i], lf = (float) img[li], rf = (float) img[ri];
        float b = (lf + cf * 2.f + rf) * 0.25f;
        float yy = b * b * 0.5f - 0.125f;
        half o = half(yy);
        memcpy(&want[i], &o, 2);
    }
    for (uint32_t i = 0; i < n; ++i) want_m[n - 1 - i] = want[i];

    int fail = 0;
    auto cmp = [&](const char *what, const std::vector<uint16_t> &got, const std::vector<uint16_t> &ref) {
        size_t bad = 0;
        for (size_t i = 0; i < ref.size(); ++i) bad += got[i] != ref[i];
        printf("%-10s n=%zu mismatches=%zu\n", what, ref.size(), bad);
        fail |= bad != 0;
    };
    cmp("filter", bits_of(out), want);
    cmp("scatter", bits_of(mirrored), want_m);

    /* literal: half(double) rounds through float (1 + 2^-11 + 2^-30 -> 0x3c00) */
    HalfC lit = HalfC(1.0 + 0x1p-11 + 0x1p-30);
    half lv = lit.coeff(0);
    uint16_t lb; memcpy(&lb, &lv, 2);
    printf("literal    0x%04x\n", lb);
    fail |= lb != 0x3c00;

    /* bit casts */
    std::vector<uint16_t> src(4099);
    for (size_t i = 0; i < src.size(); ++i) src[i] = (uint16_t) (i * 40503u);
    UInt16C u = UInt16C::copy(src.data(), src.size());
    HalfC hb = reinterpret_array<HalfC>(u);
    cmp("bitcast", bits_of(hb), src);
    std::vector<uint16_t> back(src.size());
    UInt16C ub = reinterpret_array<UInt16C>(hb);
    ub.eval();
    cuda_memcpy_from_device(back.data(), ub.data(), back.size() * 2);
    cmp("bitcast2", back, src);

    printf(fail ? "half_check FAILED\n" : "half_check ok\n");
    return fail;
}
