/* The native Float32 carlson_rf, carlson_rd and carlson_rc of include/enoki/cuda.h (the overloads of
   Array<CUDAArray<float>, 3> and Array<CUDAArray<float>, 2>) against the reference's generic bodies in
   include/enoki/special.h, which carlson_rf<Array<FloatC, 3>>(xyz) ... with explicit template arguments still record one
   primitive node per loop pass, with one evaluation and synchronisation per pass.  Both run on the device and are
   compared there, bit for bit:
   - the cross product of special values (negative, zero, denormal, tiny, huge, infinite, NaN), 2^24 random valid triples
     or pairs over 2^-40 ... 2^40, and 2^24 random bit patterns;
   - carlson_rf / carlson_rd with y computed just before (x is then loaded by the instruction), and carlson_rc in both
     operand orders (the reversed form);
   - comp_ellint_1 / 2 and ellint_1 / 2, which take the overloads, against the same templates instantiated with a
     derived vector type, which the overloads do not match.
   Then the sweeps: native comp_ellint_1(k) is exactly one sweep (the traced count is printed beside it), and
   DiffArray<CUDAArray<float>>, CUDAArray<double> and a type derived from Array keep the templates (more than one sweep).
   Built with -DNDEBUG: the templates' assert on the argument domain would abort on the invalid inputs.  Prints one line
   per check and "ell_check ok" when every mismatch count is 0.  Written from scratch. */
#include <enoki/autodiff.h>
#include <enoki/cuda.h>
#include <enoki/special.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

using namespace enoki;
using FloatC = CUDAArray<float>;
using UInt32C = CUDAArray<uint32_t>;
using DoubleC = CUDAArray<double>;
using FloatD = DiffArray<FloatC>;
using V2 = Array<FloatC, 2>;
using V3 = Array<FloatC, 3>;

/* a vector type derived from Array's base, as applications define their own Vector / Point types */
template <typename Value_> struct Vec3 : StaticArrayImpl<Value_, 3, false, Vec3<Value_>> {
    using Base = StaticArrayImpl<Value_, 3, false, Vec3<Value_>>;
    using ArrayType = Vec3;
    using MaskType = Mask<Value_, 3>;
    template <typename T> using ReplaceValue = Vec3<T>;
    ENOKI_ARRAY_IMPORT(Base, Vec3)
};

static size_t mismatches(const FloatC &a, const FloatC &b) {
    return count(neq(reinterpret_array<UInt32C>(a), reinterpret_array<UInt32C>(b)));
}

static uint64_t sweeps() { ek_stats st; ek_stats_get(&st); return st.sweep_launches; }

static float fbits(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

static FloatC native3(int f, const FloatC &x, const FloatC &y, const FloatC &z) {
    return f == 0 ? carlson_rf(V3(x, y, z)) : carlson_rd(V3(x, y, z));
}
static FloatC traced3(int f, const FloatC &x, const FloatC &y, const FloatC &z) {
    return f == 0 ? carlson_rf<V3>(V3(x, y, z)) : carlson_rd<V3>(V3(x, y, z));
}

/* special.h's complete and incomplete integrals as templates: instantiated with Vec3, which the overloads of
   Array<CUDAArray<float>, 3> do not match, every carlson_rf / carlson_rd they call is special.h's template.  (For
   |phi| > pi / 2, ellint_* adds comp_ellint_*(k), which it calls with its default arguments: that term takes the
   overloads in both forms, and comp_ellint_* is compared with its template on its own.) */
static FloatC traced_comp(int f, const FloatC &k) {
    if (f == 0) return comp_ellint_1<FloatC, FloatC, float, Vec3<FloatC>>(k);
    return comp_ellint_2<FloatC, FloatC, float, Vec3<FloatC>>(k);
}
static FloatC traced_incomplete(int f, const FloatC &phi, const FloatC &k) {
    if (f == 0) return ellint_1<FloatC, FloatC, FloatC, float, Vec3<FloatC>>(phi, k);
    return ellint_2<FloatC, FloatC, FloatC, float, Vec3<FloatC>>(phi, k);
}

int main() {
    int fail = 0;
    std::mt19937_64 rng(20261018);
    auto bits = [&]() { return fbits((uint32_t) rng()); };
    auto lg = [&]() { return std::exp2(-40.f + 80.f * (float) ((rng() >> 40) * 0x1p-24)); };
    auto uni = [&](float lo, float hi) { return lo + (hi - lo) * (float) ((rng() >> 40) * 0x1p-24); };

    std::vector<float> sp;
    {
        const float pos[] = { 0.f, 1e-45f, 1e-40f, 1.17549435e-38f, 1e-30f, 1e-4f, 0.5f, 0.99999994f, 1.f, 1.0000001f,
                              2.f, 3.f, 1e4f, 1e30f, 3.4028235e38f, fbits(0x7f800000u), fbits(0x7fc00000u) };
        for (float v : pos) { sp.push_back(v); sp.push_back(-v); }
    }
    const size_t S = sp.size();
    const char *sets[3] = { "special cross product", "2^24 random valid arguments", "2^24 random bit patterns" };
    const char *names[2] = { "carlson_rf", "carlson_rd" };
    for (int s = 0; s < 3; ++s) {
        const size_t n = s == 0 ? S * S * S : (1u << 24);
        std::vector<float> xs(n), ys(n), zs(n);
        for (size_t i = 0; i < n; ++i) {
            if (s == 0) { xs[i] = sp[i / (S * S)]; ys[i] = sp[(i / S) % S]; zs[i] = sp[i % S]; }
            else if (s == 1) { xs[i] = (i % 10 == 0) ? 0.f : lg(); ys[i] = lg(); zs[i] = lg(); }
            else { xs[i] = bits(); ys[i] = bits(); zs[i] = bits(); }
        }
        FloatC x = FloatC::copy(xs.data(), n), y = FloatC::copy(ys.data(), n), z = FloatC::copy(zs.data(), n);
        for (int f = 0; f < 2; ++f) {
            size_t bad = mismatches(native3(f, x, y, z), traced3(f, x, y, z));
            /* y computed in the same sweep: the accumulator holds y, the instruction loads x itself */
            FloatC y1 = y * 1.f;
            size_t bad1 = mismatches(native3(f, x, y1, z), traced3(f, x, y1, z));
            printf("%-10s %s: mismatches=%zu, y computed: mismatches=%zu\n", names[f], sets[s], bad, bad1);
            fail |= bad != 0 || bad1 != 0;
        }
        /* carlson_rc on (x, y), and with y computed (the reversed form) */
        const size_t m = s == 0 ? S * S : n;
        FloatC cx = x;
        if (s == 0) {
            std::vector<float> px(m), py(m);
            for (size_t i = 0; i < m; ++i) { px[i] = sp[i / S]; py[i] = sp[i % S]; }
            cx = FloatC::copy(px.data(), m);
            y = FloatC::copy(py.data(), m);
        }
        FloatC y1 = y * 1.f;
        size_t bad = mismatches(carlson_rc(V2(cx, y)), carlson_rc<V2>(V2(cx, y)));
        size_t badr = mismatches(carlson_rc(V2(cx, y1)), carlson_rc<V2>(V2(cx, y1)));
        printf("%-10s %s: mismatches=%zu, reversed: mismatches=%zu\n", "carlson_rc", sets[s], bad, badr);
        fail |= bad != 0 || badr != 0;
    }

    /* the complete and incomplete integrals through the overloads */
    {
        const size_t n = 1u << 22;
        std::vector<float> ks(n), ps(n);
        for (size_t i = 0; i < n; ++i) { ks[i] = uni(-1.f, 1.f); ps[i] = uni(-1.5f, 1.5f); }
        FloatC k = FloatC::copy(ks.data(), n), phi = FloatC::copy(ps.data(), n);
        size_t b1 = mismatches(comp_ellint_1(k), traced_comp(0, k)), b2 = mismatches(comp_ellint_2(k), traced_comp(1, k));
        size_t b3 = mismatches(ellint_1(phi, k), traced_incomplete(0, phi, k));
        size_t b4 = mismatches(ellint_2(phi, k), traced_incomplete(1, phi, k));
        for (size_t i = 0; i < n; ++i) ps[i] = uni(-8.f, 8.f);
        FloatC phi2 = FloatC::copy(ps.data(), n);
        size_t b5 = mismatches(ellint_1(phi2, k), traced_incomplete(0, phi2, k));
        size_t b6 = mismatches(ellint_2(phi2, k), traced_incomplete(1, phi2, k));
        printf("comp_ellint_1: mismatches=%zu, comp_ellint_2: mismatches=%zu\n", b1, b2);
        printf("ellint_1 |phi| <= 1.5: mismatches=%zu, |phi| <= 8: mismatches=%zu\n", b3, b5);
        printf("ellint_2 |phi| <= 1.5: mismatches=%zu, |phi| <= 8: mismatches=%zu\n", b4, b6);
        fail |= (b1 | b2 | b3 | b4 | b5 | b6) != 0;

        /* sweeps per call */
        ek_sync();
        uint64_t s0 = sweeps();
        FloatC r = comp_ellint_1(k);
        r.eval();
        ek_sync();
        uint64_t s1 = sweeps();
        FloatC t = traced_comp(0, k);
        t.eval();
        ek_sync();
        uint64_t s2 = sweeps();
        printf("sweeps of comp_ellint_1(k): native %llu, traced %llu\n", (unsigned long long) (s1 - s0),
               (unsigned long long) (s2 - s1));
        fail |= s1 - s0 != 1 || s2 - s1 <= 1;
    }

    /* the templates stay where the overloads do not match exactly */
    {
        const size_t n = 1u << 16;
        std::vector<float> xs(n), ys(n), zs(n);
        for (size_t i = 0; i < n; ++i) { xs[i] = lg(); ys[i] = lg(); zs[i] = lg(); }
        FloatC x = FloatC::copy(xs.data(), n), y = FloatC::copy(ys.data(), n), z = FloatC::copy(zs.data(), n);
        auto count_sweeps = [&](auto &&fn) {
            ek_sync();
            uint64_t a = sweeps();
            auto r = fn();
            cuda_eval();
            ek_sync();
            return sweeps() - a;
        };
        uint64_t native = count_sweeps([&]() { return carlson_rf(V3(x, y, z)); });
        uint64_t diff = count_sweeps([&]() { return carlson_rf(Array<FloatD, 3>(FloatD(x), FloatD(y), FloatD(z))); });
        uint64_t wide = count_sweeps([&]() {
            return carlson_rf(Array<DoubleC, 3>(DoubleC(x), DoubleC(y), DoubleC(z)));
        });
        uint64_t derived = count_sweeps([&]() { return carlson_rf(Vec3<FloatC>(x, y, z)); });
        uint64_t rc_diff = count_sweeps([&]() { return carlson_rc(Array<FloatD, 2>(FloatD(x), FloatD(y))); });
        printf("sweeps of carlson_rf: Array<CUDAArray<float>, 3> %llu, Array<DiffArray<CUDAArray<float>>, 3> %llu, "
               "Array<CUDAArray<double>, 3> %llu, derived Vec3<CUDAArray<float>> %llu; carlson_rc on DiffArray %llu\n",
               (unsigned long long) native, (unsigned long long) diff, (unsigned long long) wide,
               (unsigned long long) derived, (unsigned long long) rc_diff);
        fail |= native != 1 || diff <= 1 || wide <= 1 || derived <= 1 || rc_diff <= 1;
        size_t bad = mismatches(carlson_rf(Vec3<FloatC>(x, y, z)), carlson_rf(V3(x, y, z)));
        printf("derived Vec3 (template) against the overload: mismatches=%zu\n", bad);
        fail |= bad != 0;
    }
    if (!fail) printf("ell_check ok\n");
    return fail;
}
