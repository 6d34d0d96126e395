/* The native Float32 trigonometric operations of include/enoki/cuda.h (CUDAArray<float>::tan_() ... atan2_()) against
   the reference's generic bodies, which array_math.h's macros name enoki::detail::tan_impl ... atan2_impl: those record
   the same formula one primitive node at a time.  Both run on the device and are compared there, bit for bit:
     - tan, cot, asin, acos, atan: every one of the 2^32 Float32 bit patterns, in chunks of 2^26;
     - atan2: the cross product of special values (signed zeros, denormals, +-1, infinities, NaN, |y| = |x|) and 2^26
       pairs of random bit patterns.
   Then DiffArray<CUDAArray<float>> gradients of a program that uses all six, against the reference CPU tape
   (DiffArray<DynamicArray<Packet<float, 8>>>), within the bound of the CPU path's rcp / rsqrt (rcpps / rsqrtps + one
   Newton step; the backend rounds both correctly).
   Prints one line per check and "trig_check ok" when every mismatch count is 0.  Written from scratch. */
#include <enoki/autodiff.h>
#include <enoki/cuda.h>
#include <enoki/dynamic.h>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

using namespace enoki;
using FloatC = CUDAArray<float>;
using UInt32C = CUDAArray<uint32_t>;
using FloatX = DynamicArray<Packet<float, 8>>;

static size_t mismatches(const FloatC &a, const FloatC &b) {
    return count(neq(reinterpret_array<UInt32C>(a), reinterpret_array<UInt32C>(b)));
}

/* a bijective mix of the element index (so that random pairs need no host data) */
static UInt32C hash(UInt32C v, uint32_t seed) {
    v = v * 0x9E3779B1u + seed;
    v = v ^ sr<16>(v); v = v * 0x85EBCA6Bu;
    v = v ^ sr<13>(v); v = v * 0xC2B2AE35u;
    return v ^ sr<16>(v);
}

/* one function per tape (f = 0 ... 5: tan, cot, asin, acos, atan, atan2), so that no sum of terms cancels and the
   comparison can be relative per element */
template <typename FloatD> std::vector<float> gradients(int f) {
    using Float = std::decay_t<decltype(detach(std::declval<const FloatD &>()))>;
    /* the same host values for both tapes (linspace() itself differs between the CPU and CUDA arrays in the last bits) */
    std::vector<float> hx(301), hy(301);
    for (int k = 0; k < 301; ++k) { hx[k] = -0.9f + (float) k * (1.85f / 300.f); hy[k] = 1.7f - (float) k * (4.f / 300.f); }
    FloatD x = FloatD(Float::copy(hx.data(), hx.size())), y = FloatD(Float::copy(hy.data(), hy.size()));
    set_requires_gradient(x); set_requires_gradient(y);
    FloatD z = f == 0 ? tan(x) : f == 1 ? cot(y) : f == 2 ? asin(x) : f == 3 ? acos(x) : f == 4 ? atan(y) : atan2(y, x);
    backward(hsum(z));
    std::vector<float> r;
    for (const Float &v : { detach(z), gradient(x), gradient(y) }) {
        std::vector<float> h(v.size());
        if constexpr (is_cuda_array_v<Float>) { v.eval(); cuda_memcpy_from_device(h.data(), v.data(), h.size() * 4); }
        else for (size_t i = 0; i < h.size(); ++i) h[i] = v.coeff(i);
        r.insert(r.end(), h.begin(), h.end());
    }
    return r;
}

int main() {
    int fail = 0;
    const uint32_t chunk = 1u << 26;
    const char *names[5] = { "tan", "cot", "asin", "acos", "atan" };
    for (int f = 0; f < 5; ++f) {
        size_t bad = 0, bad_atan2 = 0;
        for (uint64_t base = 0; base < (1ull << 32); base += chunk) {
            FloatC x = reinterpret_array<FloatC>(arange<UInt32C>(chunk) + (uint32_t) base);
            switch (f) {
                case 0: bad += mismatches(tan(x), detail::tan_impl(x)); break;
                case 1: bad += mismatches(cot(x), detail::cot_impl(x)); break;
                case 2: bad += mismatches(asin(x), detail::asin_impl(x)); break;
                case 3: bad += mismatches(acos(x), detail::acos_impl(x)); break;
                default:
                    /* atan_impl is atan2(x, 1), which itself is native now: also against the fully traced atan2 body */
                    bad += mismatches(atan(x), detail::atan_impl(x));
                    bad_atan2 += mismatches(atan(x), detail::atan2_impl(x, FloatC(1.f)));
                    break;
            }
        }
        printf("%-6s all 2^32 inputs: mismatches=%zu\n", names[f], bad);
        fail |= bad != 0;
        if (f == 4) { printf("%-6s all 2^32 inputs vs atan2_impl(x, 1): mismatches=%zu\n", "atan", bad_atan2); fail |= bad_atan2 != 0; }
    }

    /* atan2: special values x special values, then random bit patterns */
    const float inf = INFINITY, nan_ = NAN;
    std::vector<float> s = { 0.f, -0.f, 1e-45f, -1e-45f, 1.1754942e-38f, -1.1754942e-38f, 5.877472e-39f, 1.f, -1.f, 0.5f,
                             -0.5f, 2.f, -3.f, 3.4028235e38f, -3.4028235e38f, inf, -inf, nan_, -nan_ };
    std::vector<float> ys, xs;
    for (float a : s) for (float b : s) { ys.push_back(a); xs.push_back(b); }
    FloatC ya = FloatC::copy(ys.data(), ys.size()), xa = FloatC::copy(xs.data(), xs.size());
    size_t bad_s = mismatches(atan2(ya, xa), detail::atan2_impl(ya, xa));
    printf("atan2  special cross product (%zu pairs): mismatches=%zu\n", ys.size(), bad_s);
    UInt32C i = arange<UInt32C>(chunk);
    FloatC yr = reinterpret_array<FloatC>(hash(i, 1)), xr = reinterpret_array<FloatC>(hash(i, 2));
    size_t bad_r = mismatches(atan2(yr, xr), detail::atan2_impl(yr, xr));
    FloatC yu = reinterpret_array<FloatC>(hash(i, 3)), xu = select(eq(i & 1u, 0u), yu, -yu);       /* |y| = |x| */
    bad_r += mismatches(atan2(yu, xu), detail::atan2_impl(yu, xu));
    printf("atan2  2^26 random pairs + 2^26 |y| = |x| pairs: mismatches=%zu\n", bad_r);
    fail |= bad_s != 0 || bad_r != 0;

    /* gradients: this backend's tape against the reference CPU tape */
    double worst = 0;
    size_t gbad = 0, total = 0;
    for (int f = 0; f < 6; ++f) {
        std::vector<float> g = gradients<DiffArray<FloatC>>(f), c = gradients<DiffArray<FloatX>>(f);
        gbad += g.size() != c.size();
        for (size_t k = 0; k < g.size() && k < c.size(); ++k, ++total) {
            double d = std::fabs((double) g[k] - (double) c[k]), tol = 2e-6 * std::fabs((double) c[k]);
            worst = std::fmax(worst, d / (std::fabs((double) c[k]) + 1e-30));
            gbad += !(d <= tol);
        }
    }
    printf("gradients vs reference CPU tape (%zu values): outside the rcp / rsqrt bound=%zu, worst relative=%.3g\n", total, gbad, worst);
    fail |= gbad != 0;
    if (!fail) printf("trig_check ok\n");
    return fail;
}
