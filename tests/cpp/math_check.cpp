/* The native Float32 pow, frexp, hypot, dawson and erfi of include/enoki/cuda.h (the CUDAArray<float> members pow_ and
   frexp_ and the overloads of hypot, dawson and erfi) against the reference's generic bodies in
   include/enoki/array_math.h and special.h, which detail::pow_impl<FloatC> ... and the templates with explicit arguments
   still record one primitive node at a time.  Both run on the device and are compared there, bit for bit:
   - dawson, erfi and both outputs of frexp for every one of the 2^32 Float32 bit patterns (in chunks of 2^26);
   - pow and hypot, in both operand orders (the second with a computed operand: the reversed forms), on the cross
     product of special values, 2^26 random bit-pattern pairs, positive bases with exponents in [-8, 8] and operands of
     equal magnitude.
   First, a dry run (nothing launched): the unqualified calls on CUDAArray<float> are one body instruction each (frexp
   two), while DiffArray<CUDAArray<float>>, CUDAArray<double> and a mixed call such as hypot(x, 1.f) keep the traced
   bodies.  Prints one line per check and "math_check ok" when every mismatch count is 0.  Written from scratch. */
#include <enoki/autodiff.h>
#include <enoki/cuda.h>
#include <enoki/special.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

/* the dry-run listing of the library (not in the public header): malloc'd, freed by the caller */
extern "C" char *ek_debug_plan(void);

using namespace enoki;
using FloatC = CUDAArray<float>;
using UInt32C = CUDAArray<uint32_t>;
using DoubleC = CUDAArray<double>;
using FloatD = DiffArray<FloatC>;

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

static const char *bnames[2] = { "pow", "hypot" };
static const char *unames[4] = { "frexp_m", "frexp_e", "dawson", "erfi" };

/* binary function f, unqualified: the members of CUDAArray<float> through array_math.h's dispatch, and cuda.h's
   overload of hypot */
template <typename T> static T bcall(int f, const T &x, const T &y) {
    switch (f) {
        case 0: return pow(x, y);
        default: return hypot(x, y);
    }
}
static FloatC btraced(int f, const FloatC &x, const FloatC &y) {
    switch (f) {
        case 0: return detail::pow_impl<FloatC>(x, y);
        default: return hypot<FloatC, FloatC>(x, y);
    }
}
template <typename T> static T ucall(int f, const T &x) {
    switch (f) {
        case 0: return frexp(x).first;
        case 1: return frexp(x).second;
        case 2: return dawson(x);
        default: return erfi(x);
    }
}
/* erfi<FloatC> calls dawson unqualified, which finds cuda.h's overload: the reference body is spelled out here */
static FloatC utraced(int f, const FloatC &x) {
    switch (f) {
        case 0: return detail::frexp_impl<FloatC>(x).first;
        case 1: return detail::frexp_impl<FloatC>(x).second;
        case 2: return dawson<FloatC>(x);
        default: return float(M_2_SQRTPI) * dawson<FloatC>(x) * exp(x * x);
    }
}

static float fbits(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

int main() {
    int fail = 0;
    {
        const size_t n = 1 << 20;
        FloatC m = FloatC::map((void *) 0x7f0001000000ull, n), m2 = FloatC::map((void *) 0x7f0003000000ull, n);
        DoubleC md = DoubleC::map((void *) 0x7f0002000000ull, n), md2 = DoubleC::map((void *) 0x7f0004000000ull, n);
        for (int f = 0; f < 2; ++f) {
            int native, diff, wide;
            { FloatC r = bcall(f, m, m2); native = body_len(); }
            { FloatD r = bcall(f, FloatD(m), FloatD(m2)); diff = body_len(); }
            { DoubleC r = bcall(f, md, md2); wide = body_len(); }
            printf("dry run of %s: CUDAArray<float> %d, DiffArray<CUDAArray<float>> %d, CUDAArray<double> %d body "
                   "instructions\n", bnames[f], native, diff, wide);
            fail |= native != 1 || diff <= 1 || wide <= 1;
        }
        for (int f = 0; f < 4; ++f) {
            int native, diff, wide;
            { FloatC r = ucall(f, m); native = body_len(); }
            { FloatD r = ucall(f, FloatD(m)); diff = body_len(); }
            { DoubleC r = ucall(f, md); wide = body_len(); }
            printf("dry run of %s: CUDAArray<float> %d, DiffArray<CUDAArray<float>> %d, CUDAArray<double> %d body "
                   "instructions\n", unames[f], native, diff, wide);
            fail |= native != 1 || diff <= 1 || wide <= 1;
        }
        { auto r = frexp(m); int k = body_len(); printf("dry run of frexp (both outputs): %d\n", k); fail |= k != 2; }
        { FloatC r = hypot(m, 1.f); int k = body_len(); printf("dry run of hypot(x, 1.f): %d\n", k); fail |= k <= 1; }
    }

    /* unary functions: every input */
    const uint32_t chunk = 1u << 26;
    for (int f = 0; f < 4; ++f) {
        size_t bad = 0;
        for (uint64_t base = 0; base < (1ull << 32); base += chunk) {
            FloatC x = reinterpret_array<FloatC>(arange<UInt32C>(chunk) + (uint32_t) base);
            bad += mismatches(ucall(f, x), utraced(f, x));
        }
        printf("%-8s all 2^32 inputs: mismatches=%zu\n", unames[f], bad);
        fail |= bad != 0;
    }

    /* binary functions: pairs built on the host */
    std::vector<float> sp;
    {
        const float pos[] = { 0.f, 1e-45f, 1e-40f, 1.1754942e-38f, 1.17549435e-38f, 1e-30f, 1e-4f, 0.5f, 0.99999994f, 1.f,
                              1.0000001f, 1.5f, 2.f, 2.5f, 3.f, 7.f, 8.f, 10.f, 88.f, 100.f, 127.f, 128.f, 1e10f,
                              16777216.f, 3.4028235e38f, fbits(0x7f800000u), fbits(0x7fc00000u), fbits(0x7fa00000u),
                              fbits(0x7fffffffu) };
        for (float v : pos) { sp.push_back(v); sp.push_back(-v); }
    }
    std::mt19937_64 rng(20261020);
    auto bits = [&]() { return fbits((uint32_t) rng()); };
    auto uni = [&](float lo, float hi) { return lo + (hi - lo) * (float) ((rng() >> 40) * 0x1p-24); };
    const char *sets[4] = { "special cross product", "2^26 random bit patterns", "positive bases", "equal magnitudes" };
    for (int s = 0; s < 4; ++s) {
        size_t bad[2][2] = {};
        const size_t batches = s == 1 ? 4 : 1, n = s == 0 ? sp.size() * sp.size() : s == 1 ? (1u << 24) : (1u << 22);
        for (size_t batch = 0; batch < batches; ++batch) {
            std::vector<float> xs(n), ys(n);
            for (size_t i = 0; i < n; ++i) {
                if (s == 0) { xs[i] = sp[i / sp.size()]; ys[i] = sp[i % sp.size()]; }
                else if (s == 1) { xs[i] = bits(); ys[i] = bits(); }
                else if (s == 3) { xs[i] = uni(-1e3f, 1e3f); ys[i] = (i & 1) ? -xs[i] : xs[i]; }
                else { xs[i] = uni(0.f, 10.f); ys[i] = uni(-8.f, 8.f); }
            }
            FloatC x = FloatC::copy(xs.data(), n), y = FloatC::copy(ys.data(), n);
            for (int f = 0; f < 2; ++f) {
                bad[f][0] += mismatches(bcall(f, x, y), btraced(f, x, y));
                /* the operands swapped, the second one computed in the same sweep: the native call then runs the
                   reversed form (the accumulator holds the second operand) */
                FloatC x1 = x * 1.f;
                bad[f][1] += mismatches(bcall(f, y, x1), btraced(f, y, x1));
            }
        }
        for (int f = 0; f < 2; ++f) {
            printf("%-6s %s: mismatches=%zu, swapped and reversed: mismatches=%zu\n", bnames[f], sets[s], bad[f][0], bad[f][1]);
            fail |= bad[f][0] != 0 || bad[f][1] != 0;
        }
    }
    if (!fail) printf("math_check ok\n");
    return fail;
}
