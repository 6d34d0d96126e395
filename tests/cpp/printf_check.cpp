/* cuda_printf through the reference's own template (array_router.h:971-975) over this repo's enoki::CUDAArray<T>.
   stdout carries exactly the printed lines (tests/test_gpu_printf.py compares them with the C library's snprintf);
   the checks of this program report on stderr.  Built by tests/cpp/printf_check.mk; exit code 0 = all checks passed. */
#include <enoki/cuda.h>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>

using namespace enoki;
using FloatC = CUDAArray<float>;
using UInt32C = CUDAArray<uint32_t>;

static int failures = 0;
#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "CHECK failed: %s (%s:%d)\n", #cond, __FILE__, __LINE__); ++failures; } } while (0)

template <typename... Args> static std::string rejected(const char *fmt, const Args &... args) {
    try { cuda_printf(fmt, args...); } catch (const std::runtime_error &e) { return e.what(); }
    return "";
}

int main() {
    if (ek_device_count() == 0) { fprintf(stderr, "no CUDA device\n"); return 2; }

    UInt32C i = arange<UInt32C>(11);
    FloatC x = FloatC(i) * 0.125f;
    cuda_printf("i=%u x=%f y=%.4e\n", i, x, x * x + 1.f);
    cuda_eval();

    cuda_printf("scalar %u\n", UInt32C(7));
    cuda_eval();

    cuda_printf("no arguments\n");
    cuda_eval();

    cuda_printf("%u %g\n", arange<UInt32C>(3) * 3u, FloatC(0.5f));
    cuda_eval();

    /* rejected prints throw and record nothing */
    CHECK(rejected("%s\n", x).find("'%s'") != std::string::npos);
    CHECK(rejected("%d\n", x).find("f32") != std::string::npos);
    CHECK(rejected("%f %f %f %f\n", x, x, x, x) == "cuda_trace_print(): at most 3 variables can be printed at once!");
    CHECK(rejected("%u\n", UInt32C()).find("uninitialized") != std::string::npos);
    fflush(stdout);
    cuda_eval();

    /* the printed arrays are untouched */
    CHECK(x.coeff(10) == 1.25f && i.coeff(10) == 10u);
    if (failures) { fprintf(stderr, "%d check(s) failed\n", failures); return 1; }
    fprintf(stderr, "all checks passed\n");
    return 0;
}
