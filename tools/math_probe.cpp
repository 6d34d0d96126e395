/* math_probe: the sweep kernel time of the native Float32 pow, frexp, hypot, dawson and erfi (the
   CUDAArray<float> members and overloads of include/enoki/cuda.h) against the traced bodies of array_math.h and
   special.h (detail::pow_impl<FloatC> ... and the templates with explicit arguments, one recorded node per primitive;
   erfi's is M_2_SQRTPI * dawson<FloatC>(x) * exp(x * x)), at 2^26 elements.  pow is measured with an array exponent and
   with the scalar one of pow(x, 2.2f), whose native form reads the exponent from the uniform pool.  The two forms
   alternate, the device time of every launch is taken with CUDA events (ek_set_timing), and the body length of each form
   comes from the dry run (ek_debug_plan).  Prints one JSON object with the card's name and power limit.
   Build: make -C tools math_probe (reference headers needed, like c5_bench). */
#include <enoki/cuda.h>
#include <enoki/special.h>
#include <dlfcn.h>
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

/* the dry-run listing of the library (not in the public header): malloc'd, freed by the caller */
extern "C" char *ek_debug_plan(void);

using namespace enoki;
using FloatC = CUDAArray<float>;
using UInt32C = CUDAArray<uint32_t>;

static FloatC input(size_t n, uint32_t seed, float lo, float hi) {
    UInt32C i = arange<UInt32C>(n) * 0x9E3779B1u + seed;
    i = i ^ sr<15>(i); i = i * 0x85EBCA6Bu; i = i ^ sr<13>(i);
    FloatC u = FloatC(sr<8>(i)) * (1.f / 16777216.f);
    FloatC r = fmadd(u, hi - lo, lo);
    r.eval();
    return r;
}

/* body instructions of the pending sweeps (dry run: nothing is launched) */
static int body_len() {
    char *p = ek_debug_plan();
    if (!p) return -1;
    int n = 0;
    for (const char *s = p; (s = strstr(s, "\n  body ")); ++s) ++n;
    free(p);
    return n;
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

template <typename F1, typename F2> static void measure(const char *name, F1 native, F2 traced, int reps) {
    int len[2];
    double best[2] = { 1e30, 1e30 }, sum[2] = { 0, 0 };
    auto run = [&](int form, bool dry) {
        if (form) { auto r = traced(); if (dry) len[form] = body_len(); cuda_eval(); }
        else { auto r = native(); if (dry) len[form] = body_len(); cuda_eval(); }
    };
    for (int form = 0; form < 2; ++form) { run(form, true); cuda_sync(); }   /* warm-up, and the dry-run lengths */
    for (int k = 0; k < reps; ++k) {
        for (int form = 0; form < 2; ++form) {
            cuda_sync();
            ek_set_timing(1); ek_stats_reset();
            run(form, false); cuda_sync();
            ek_stats st; ek_stats_get(&st);
            ek_set_timing(0);
            best[form] = std::min(best[form], (double) st.total_kernel_ms);
            sum[form] += st.total_kernel_ms;
        }
    }
    printf(", \"%s\": {\"native_body\": %d, \"traced_body\": %d, \"native_ms_min\": %.4f, \"traced_ms_min\": %.4f, "
           "\"native_ms_mean\": %.4f, \"traced_ms_mean\": %.4f, \"speedup_min\": %.2f}", name, len[0], len[1],
           best[0], best[1], sum[0] / reps, sum[1] / reps, best[1] / best[0]);
}

int main(int argc, char **argv) {
    const size_t n = (size_t) 1 << 26;
    const int reps = argc > 1 ? atoi(argv[1]) : 10;
    FloatC x = input(n, 1, 0.f, 10.f), y = input(n, 2, -8.f, 8.f), s = input(n, 3, -100.f, 100.f),
           d = input(n, 5, -6.f, 6.f);
    cuda_sync();
    char name[96];
    double watts;
    card(name, sizeof(name), &watts);
    printf("{\"device\": \"%s\", \"power_limit_w\": %.0f, \"elements\": %zu, \"reps\": %d", name, watts, n, reps);
    measure("pow", [&] { return pow(x, y); }, [&] { return detail::pow_impl<FloatC>(x, y); }, reps);
    measure("pow_scalar", [&] { return pow(x, 2.2f); }, [&] { return detail::pow_impl<FloatC>(x, FloatC(2.2f)); }, reps);
    measure("frexp", [&] { return frexp(s); }, [&] { return detail::frexp_impl<FloatC>(s); }, reps);
    measure("hypot", [&] { return hypot(s, y); }, [&] { return hypot<FloatC, FloatC>(s, y); }, reps);
    measure("dawson", [&] { return dawson(d); }, [&] { return dawson<FloatC>(d); }, reps);
    measure("erfi", [&] { return erfi(d); }, [&] { return float(M_2_SQRTPI) * dawson<FloatC>(d) * exp(d * d); }, reps);
    printf("}\n");
    return 0;
}
