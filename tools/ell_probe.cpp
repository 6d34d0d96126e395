/* ell_probe: the time of the native Float32 carlson_rf, carlson_rd and carlson_rc (the overloads of
   Array<CUDAArray<float>, N> in include/enoki/cuda.h) against special.h's traced bodies (the templates with explicit
   arguments: one recorded pass of the duplication loop per evaluation, with one synchronisation each), and of
   comp_ellint_1 / 2 and ellint_1 / 2, which take the overloads, against the same templates instantiated with a derived
   vector type (which the overloads do not match), at 2^26 elements; and carlson_rj with its inner carlson_rc native (the overload) against traced.  The traced forms
   synchronise on their own, so each form is timed with the host clock around work that ends in ek_sync(); the two forms
   alternate.  Reports the sweeps each call launches, and the card's name and power limit, as one JSON object.
   Build: make -C tools ell_probe (reference headers needed, like c5_bench). */
#include <enoki/cuda.h>
#include <enoki/special.h>
#include <dlfcn.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

using namespace enoki;
using FloatC = CUDAArray<float>;
using UInt32C = CUDAArray<uint32_t>;
using V2 = Array<FloatC, 2>;
using V3 = Array<FloatC, 3>;
using V4 = Array<FloatC, 4>;

/* vector types derived from Array's base, as applications define their own: the overloads of carlson_rf / carlson_rd /
   carlson_rc do not match them, so special.h's functions instantiated with them record the templates */
template <typename Value_> struct Vec3 : StaticArrayImpl<Value_, 3, false, Vec3<Value_>> {
    using Base = StaticArrayImpl<Value_, 3, false, Vec3<Value_>>;
    using ArrayType = Vec3;
    using MaskType = Mask<Value_, 3>;
    template <typename T> using ReplaceValue = Vec3<T>;
    ENOKI_ARRAY_IMPORT(Base, Vec3)
};
template <typename Value_> struct Vec2 : StaticArrayImpl<Value_, 2, false, Vec2<Value_>> {
    using Base = StaticArrayImpl<Value_, 2, false, Vec2<Value_>>;
    using ArrayType = Vec2;
    using MaskType = Mask<Value_, 2>;
    template <typename T> using ReplaceValue = Vec2<T>;
    ENOKI_ARRAY_IMPORT(Base, Vec2)
};

static FloatC input(size_t n, uint32_t seed, float lo, float hi) {
    UInt32C i = arange<UInt32C>(n) * 0x9E3779B1u + seed;
    i = i ^ sr<15>(i); i = i * 0x85EBCA6Bu; i = i ^ sr<13>(i);
    FloatC u = FloatC(sr<8>(i)) * (1.f / 16777216.f);
    FloatC r = fmadd(u, hi - lo, lo);
    r.eval();
    return r;
}

/* the name and enforced power limit (watts) of device 0, read through NVML ("?" and -1 where it is not available) */
static void card(char *name, unsigned len, double *watts) {
    strcpy(name, "?");
    *watts = -1;
    void *h = dlopen("libnvidia-ml.so.1", RTLD_NOW);
    if (!h) return;
    auto init = (int (*)()) dlsym(h, "nvmlInit_v2");
    auto handle = (int (*)(unsigned, void **)) dlsym(h, "nvmlDeviceGetHandleByIndex_v2");
    auto get_name = (int (*)(void *, char *, unsigned)) dlsym(h, "nvmlDeviceGetName");
    auto limit = (int (*)(void *, unsigned *)) dlsym(h, "nvmlDeviceGetEnforcedPowerLimit");
    auto shutdown = (int (*)()) dlsym(h, "nvmlShutdown");
    void *dev = nullptr;
    unsigned mw = 0;
    if (init && handle && get_name && limit && init() == 0) {
        if (handle(0, &dev) == 0) {
            if (get_name(dev, name, len) != 0) strcpy(name, "?");
            if (limit(dev, &mw) == 0) *watts = mw / 1000.0;
        }
        if (shutdown) shutdown();
    }
    dlclose(h);
}

static uint64_t sweeps() { ek_stats st; ek_stats_get(&st); return st.sweep_launches; }

template <typename F1, typename F2> static void measure(const char *name, F1 native, F2 traced, int reps) {
    double best[2] = { 1e30, 1e30 }, sum[2] = { 0, 0 };
    uint64_t launches[2] = { 0, 0 };
    auto run = [&](int form) {
        ek_sync();
        uint64_t s0 = sweeps();
        auto t0 = std::chrono::steady_clock::now();
        if (form) { FloatC r = traced(); r.eval(); } else { FloatC r = native(); r.eval(); }
        ek_sync();
        double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        launches[form] = sweeps() - s0;
        return ms;
    };
    for (int form = 0; form < 2; ++form) run(form);          /* warm-up */
    for (int k = 0; k < reps; ++k) {
        for (int form = 0; form < 2; ++form) {
            double ms = run(form);
            best[form] = std::min(best[form], ms);
            sum[form] += ms;
        }
    }
    printf(", \"%s\": {\"native_sweeps\": %llu, \"traced_sweeps\": %llu, \"native_ms_min\": %.3f, \"traced_ms_min\": %.3f, "
           "\"native_ms_mean\": %.3f, \"traced_ms_mean\": %.3f, \"speedup_min\": %.2f}", name,
           (unsigned long long) launches[0], (unsigned long long) launches[1], best[0], best[1], sum[0] / reps,
           sum[1] / reps, best[1] / best[0]);
    fflush(stdout);
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

int main(int argc, char **argv) {
    const size_t n = (size_t) 1 << 26;
    const int reps = argc > 1 ? atoi(argv[1]) : 5;
    FloatC x = input(n, 1, 0.f, 4.f), y = input(n, 2, 0.01f, 4.f), z = input(n, 3, 0.01f, 4.f),
           k = input(n, 4, -0.99f, 0.99f), phi = input(n, 5, -1.5f, 1.5f);
    ek_sync();
    char name[96];
    double watts;
    card(name, sizeof(name), &watts);
    printf("{\"device\": \"%s\", \"power_limit_w\": %.0f, \"elements\": %zu, \"reps\": %d", name, watts, n, reps);
    measure("carlson_rf", [&] { return carlson_rf(V3(x, y, z)); }, [&] { return carlson_rf<V3>(V3(x, y, z)); }, reps);
    measure("carlson_rd", [&] { return carlson_rd(V3(x, y, z)); }, [&] { return carlson_rd<V3>(V3(x, y, z)); }, reps);
    measure("carlson_rc", [&] { return carlson_rc(V2(x, y)); }, [&] { return carlson_rc<V2>(V2(x, y)); }, reps);
    measure("comp_ellint_1", [&] { return comp_ellint_1(k); }, [&] { return traced_comp(0, k); }, reps);
    measure("comp_ellint_2", [&] { return comp_ellint_2(k); }, [&] { return traced_comp(1, k); }, reps);
    measure("ellint_1", [&] { return ellint_1(phi, k); }, [&] { return traced_incomplete(0, phi, k); }, reps);
    measure("ellint_2", [&] { return ellint_2(phi, k); }, [&] { return traced_incomplete(1, phi, k); }, reps);
    /* carlson_rj's own loop stays traced; its inner carlson_rc(Array<FloatC, 2>) takes the overload */
    measure("carlson_rj", [&] { return carlson_rj(V4(x, y, z, y + 1.f)); },
            [&] { return carlson_rj<V4, FloatC, Vec2<FloatC>>(V4(x, y, z, y + 1.f)); }, reps);
    printf("}\n");
    return 0;
}
