/* The native Float32 special functions of include/enoki/cuda.h (the CUDAArray<float> overloads of erf, erfc, erfinv,
   lgamma and tgamma) against the reference's generic bodies in include/enoki/special.h, which the same calls with
   explicit template arguments (erf<FloatC>(x) ...) still record one primitive node at a time.  Both run on the device
   and are compared there, bit for bit, for every one of the 2^32 Float32 bit patterns (in chunks of 2^26).
   First, a dry run (nothing launched): the unqualified calls on a CUDAArray<float> are one body instruction each, while
   DiffArray<CUDAArray<float>> and CUDAArray<double> keep the traced bodies.
   Prints one line per check and "special_check ok" when every mismatch count is 0.  Written from scratch. */
#include <enoki/autodiff.h>
#include <enoki/cuda.h>
#include <enoki/special.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>

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

static const char *names[5] = { "erf", "erfc", "erfinv", "lgamma", "tgamma" };

/* function f (0 ... 4 as in names), unqualified: overload resolution picks cuda.h's overloads for CUDAArray<float> */
template <typename T> static T call(int f, const T &x) {
    switch (f) {
        case 0: return erf(x);
        case 1: return erfc(x);
        case 2: return erfinv(x);
        case 3: return lgamma(x);
        default: return tgamma(x);
    }
}
/* the same with explicit template arguments: special.h's generic bodies.  tgamma (special.h:312) is exp(lgamma(x)) with
   lgamma called unqualified, which finds cuda.h's overload: its traced body is exp(lgamma<FloatC>(x)). */
static FloatC traced(int f, const FloatC &x) {
    switch (f) {
        case 0: return erf<FloatC>(x);
        case 1: return erfc<FloatC>(x);
        case 2: return erfinv<FloatC>(x);
        case 3: return lgamma<FloatC>(x);
        default: return exp(lgamma<FloatC>(x));
    }
}

int main() {
    int fail = 0;
    {
        const size_t n = 1 << 20;
        FloatC m = FloatC::map((void *) 0x7f0001000000ull, n);
        DoubleC md = DoubleC::map((void *) 0x7f0002000000ull, n);
        for (int f = 0; f < 5; ++f) {
            int native, diff, wide;
            { FloatC r = call(f, m); native = body_len(); }
            { FloatD r = call(f, FloatD(m)); diff = body_len(); }
            { DoubleC r = call(f, md); wide = body_len(); }
            printf("dry run of %s: CUDAArray<float> %d, DiffArray<CUDAArray<float>> %d, CUDAArray<double> %d body "
                   "instructions\n", names[f], native, diff, wide);
            fail |= native != 1 || diff <= 1 || wide <= 1;
        }
    }
    const uint32_t chunk = 1u << 26;
    for (int f = 0; f < 5; ++f) {
        size_t bad = 0;
        for (uint64_t base = 0; base < (1ull << 32); base += chunk) {
            FloatC x = reinterpret_array<FloatC>(arange<UInt32C>(chunk) + (uint32_t) base);
            bad += mismatches(call(f, x), traced(f, x));
        }
        printf("%-8s all 2^32 inputs: mismatches=%zu\n", names[f], bad);
        fail |= bad != 0;
    }
    if (!fail) printf("special_check ok\n");
    return fail;
}
