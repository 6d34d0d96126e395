/* trig_probe: the sweep kernel time of the native Float32 tan / cot / asin / acos / atan / atan2 against array_math.h's
   traced bodies (enoki::detail::*_impl, one recorded node per primitive), and of the spherical-coordinates pair
   theta = acos(z), phi = atan2(y, x), at 2^26 elements.  The two forms alternate, the device time of every launch is
   taken with CUDA events (ek_set_timing), and the body length of each form comes from the dry run (ek_debug_plan).
   Prints one JSON object.  Build: make -C tools trig_probe (reference headers needed, like c5_bench). */
#include <enoki/cuda.h>
#include <algorithm>
#include <functional>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

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

template <typename Fn> static void measure(const char *name, bool first, Fn &&native, Fn &&traced, int reps) {
    int len[2];
    double best[2] = { 1e30, 1e30 }, sum[2] = { 0, 0 };
    for (int form = 0; form < 2; ++form) {           /* warm-up, and the dry-run lengths */
        FloatC r = form ? traced() : native();
        len[form] = body_len();
        r.eval(); cuda_sync();
    }
    for (int k = 0; k < reps; ++k) {
        for (int form = 0; form < 2; ++form) {
            FloatC r = form ? traced() : native();
            cuda_sync();
            ek_set_timing(1); ek_stats_reset();
            r.eval(); cuda_sync();
            ek_stats st; ek_stats_get(&st);
            ek_set_timing(0);
            best[form] = std::min(best[form], (double) st.total_kernel_ms);
            sum[form] += st.total_kernel_ms;
        }
    }
    printf("%s\"%s\": {\"native_body\": %d, \"traced_body\": %d, \"native_ms_min\": %.4f, \"traced_ms_min\": %.4f, "
           "\"native_ms_mean\": %.4f, \"traced_ms_mean\": %.4f}", first ? "" : ", ", name, len[0], len[1],
           best[0], best[1], sum[0] / reps, sum[1] / reps);
}

int main(int argc, char **argv) {
    const size_t n = (size_t) 1 << 26;
    const int reps = argc > 1 ? atoi(argv[1]) : 10;
    FloatC x = input(n, 1, -3.f, 3.f), y = input(n, 2, -3.f, 3.f), z = input(n, 3, -1.f, 1.f);
    cuda_sync();
    printf("{\"elements\": %zu, \"reps\": %d, ", n, reps);
    using F = std::function<FloatC()>;
    measure("tan", true, F([&] { return tan(x); }), F([&] { return detail::tan_impl(x); }), reps);
    measure("cot", false, F([&] { return cot(x); }), F([&] { return detail::cot_impl(x); }), reps);
    measure("asin", false, F([&] { return asin(z); }), F([&] { return detail::asin_impl(z); }), reps);
    measure("acos", false, F([&] { return acos(z); }), F([&] { return detail::acos_impl(z); }), reps);
    measure("atan", false, F([&] { return atan(x); }), F([&] { return detail::atan2_impl(x, FloatC(1.f)); }), reps);
    measure("atan2", false, F([&] { return atan2(y, x); }), F([&] { return detail::atan2_impl(y, x); }), reps);
    measure("theta_phi", false, F([&] { return acos(z) + atan2(y, x); }),
            F([&] { return detail::acos_impl(z) + detail::atan2_impl(y, x); }), reps);
    printf("}\n");
    return 0;
}
