/* The native Float32 hyperbolic functions and cbrt of include/enoki/cuda.h (CUDAArray<float>::sinh_() ... cbrt_(),
   sincosh_()) against the reference's generic bodies, which array_math.h's macros name enoki::detail::sinh_impl ...
   cbrt_impl and sincosh_impl: those record the same formula one primitive node at a time.  Both run on the device and
   are compared there, bit for bit, for every one of the 2^32 Float32 bit patterns (in chunks of 2^26), both outputs of
   sincosh included.
   Then DiffArray<CUDAArray<float>> gradients of each function, against the reference CPU tape
   (DiffArray<DynamicArray<Packet<float, 8>>>), within the bound of the CPU path's rcp / rsqrt (rcpps / rsqrtps + one
   Newton step; the backend rounds both correctly).
   First, a dry run (nothing launched): sinh of a CUDAArray<float> and of a DiffArray<CUDAArray<float>> is one body
   instruction, while CUDAArray<double> keeps the traced body.
   Prints one line per check and "hyp_check ok" when every mismatch count is 0.  Written from scratch. */
#include <enoki/autodiff.h>
#include <enoki/cuda.h>
#include <enoki/dynamic.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

/* the dry-run listing of the library (not in the public header): malloc'd, freed by the caller */
extern "C" char *ek_debug_plan(void);

using namespace enoki;
using FloatC = CUDAArray<float>;
using UInt32C = CUDAArray<uint32_t>;
using FloatX = DynamicArray<Packet<float, 8>>;

static size_t mismatches(const FloatC &a, const FloatC &b) {
    return count(neq(reinterpret_array<UInt32C>(a), reinterpret_array<UInt32C>(b)));
}

/* body instructions of the pending sweeps */
static int body_len() {
    char *p = ek_debug_plan();
    if (!p) return -1;
    int n = 0;
    for (const char *s = p; (s = strstr(s, "\n  body ")); ++s) ++n;
    free(p);
    return n;
}

static const char *names[8] = { "sinh", "cosh", "tanh", "asinh", "acosh", "atanh", "cbrt", "sincosh" };

/* function f (0 ... 6 as in names) on one tape, over arguments inside its domain */
template <typename FloatD> std::vector<float> gradients(int f) {
    using Float = std::decay_t<decltype(detach(std::declval<const FloatD &>()))>;
    const float lo = f == 4 ? 1.1f : f == 5 ? -0.9f : -2.9f, hi = f == 4 ? 5.f : f == 5 ? 0.9f : 2.9f;
    std::vector<float> hx(301);          /* the same host values for both tapes */
    for (int k = 0; k < 301; ++k) hx[k] = lo + (float) k * ((hi - lo) / 300.f);
    FloatD x = FloatD(Float::copy(hx.data(), hx.size()));
    set_requires_gradient(x);
    FloatD z = f == 0 ? sinh(x) : f == 1 ? cosh(x) : f == 2 ? tanh(x) : f == 3 ? asinh(x) : f == 4 ? acosh(x)
             : f == 5 ? atanh(x) : cbrt(x);
    backward(hsum(z));
    std::vector<float> r;
    for (const Float &v : { detach(z), gradient(x) }) {
        std::vector<float> h(v.size());
        if constexpr (is_cuda_array_v<Float>) { v.eval(); cuda_memcpy_from_device(h.data(), v.data(), h.size() * 4); }
        else for (size_t i = 0; i < h.size(); ++i) h[i] = v.coeff(i);
        r.insert(r.end(), h.begin(), h.end());
    }
    return r;
}

int main() {
    int fail = 0;
    {
        const size_t n = 1 << 20;
        FloatC m = FloatC::map((void *) 0x7f0001000000ull, n);
        CUDAArray<double> md = CUDAArray<double>::map((void *) 0x7f0002000000ull, n);
        int native, diff, wide;
        { FloatC r = sinh(m); native = body_len(); }
        { DiffArray<FloatC> r = sinh(DiffArray<FloatC>(m)); diff = body_len(); }
        { CUDAArray<double> r = sinh(md); wide = body_len(); }
        printf("dry run of sinh: CUDAArray<float> %d, DiffArray<CUDAArray<float>> %d, CUDAArray<double> %d body instructions\n",
               native, diff, wide);
        fail |= native != 1 || diff != 1 || wide <= 1;
    }
    const uint32_t chunk = 1u << 26;
    for (int f = 0; f < 8; ++f) {
        size_t bad = 0, bad2 = 0;
        for (uint64_t base = 0; base < (1ull << 32); base += chunk) {
            FloatC x = reinterpret_array<FloatC>(arange<UInt32C>(chunk) + (uint32_t) base);
            switch (f) {
                case 0: bad += mismatches(sinh(x), detail::sinh_impl(x)); break;
                case 1: bad += mismatches(cosh(x), detail::cosh_impl(x)); break;
                case 2: bad += mismatches(tanh(x), detail::tanh_impl(x)); break;
                case 3: bad += mismatches(asinh(x), detail::asinh_impl(x)); break;
                case 4: bad += mismatches(acosh(x), detail::acosh_impl(x)); break;
                case 5: bad += mismatches(atanh(x), detail::atanh_impl(x)); break;
                case 6: bad += mismatches(cbrt(x), detail::cbrt_impl(x)); break;
                default: {
                    auto [s, c] = sincosh(x);
                    auto [ts, tc] = detail::sincosh_impl(x);
                    bad += mismatches(s, ts);
                    bad2 += mismatches(c, tc);
                }
            }
        }
        if (f < 7) printf("%-8s all 2^32 inputs: mismatches=%zu\n", names[f], bad);
        else printf("%-8s all 2^32 inputs: sinh mismatches=%zu, cosh mismatches=%zu\n", names[f], bad, bad2);
        fail |= bad != 0 || bad2 != 0;
    }

    /* gradients: this backend's tape against the reference CPU tape */
    double worst = 0;
    size_t gbad = 0, total = 0;
    for (int f = 0; f < 7; ++f) {
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
    if (!fail) printf("hyp_check ok\n");
    return fail;
}
