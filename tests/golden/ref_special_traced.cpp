/* Records the reference's generic single precision erf, erfc, erfinv, lgamma and tgamma (include/enoki/special.h) and
   the normal-sampling step sqrt(2) * erfinv(2u - 1) of tests/histogram.cpp on a CUDAArray<float> mapped over a fake
   device address, one primitive node at a time as they were recorded before these functions were native (the explicit
   template arguments pick special.h's templates over cuda.h's CUDAArray<float> overloads), and prints the dry run of
   each as one JSON object: {name: {"x": input variable, "out": [result variable], "plan": ek_debug_plan(), "program":
   ek_debug_program()}}.  Nothing is launched.  Built and run by tests/golden/make_golden_special.py, which stores the
   output as tests/golden/special_traced.json. */
#include <enoki/cuda.h>
#include <enoki/special.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <string>

using namespace enoki;
using FloatC = CUDAArray<float>;
extern "C" char *ek_debug_plan(void);
extern "C" char *ek_debug_program(void);

static std::string quoted(const char *s) {
    std::string r = "\"";
    for (; *s; ++s) {
        if (*s == '"' || *s == '\\') { r += '\\'; r += *s; }
        else if (*s == '\n') r += "\\n";
        else r += *s;
    }
    return r + "\"";
}

static void dump(bool first, const char *name, const FloatC &x, const FloatC &r) {
    char *plan = ek_debug_plan(), *prog = ek_debug_program();
    if (!plan || !prog) { fprintf(stderr, "%s: dry run failed\n", name); exit(1); }
    printf("%s\"%s\": {\"x\": %u, \"out\": [%u], \"plan\": %s, \"program\": %s}", first ? "" : ",\n", name, x.index_(),
           r.index_(), quoted(plan).c_str(), prog);
    free(plan); free(prog);
}

int main() {
    const size_t n = 1 << 20;
    FloatC x = FloatC::map((void *) 0x7f0001000000ull, n);
    printf("{");
    { FloatC r = erf<FloatC>(x);    dump(true, "erf", x, r); }
    { FloatC r = erfc<FloatC>(x);   dump(false, "erfc", x, r); }
    { FloatC r = erfinv<FloatC>(x); dump(false, "erfinv", x, r); }
    { FloatC r = lgamma<FloatC>(x); dump(false, "lgamma", x, r); }
    /* special.h:312 tgamma<FloatC> calls lgamma unqualified, which finds cuda.h's overload: its traced body is
       exp(lgamma<FloatC>(x)) */
    { FloatC r = exp(lgamma<FloatC>(x)); dump(false, "tgamma", x, r); }
    { FloatC r = float(M_SQRT2) * erfinv<FloatC>(2.f * x - 1.f); dump(false, "normal", x, r); }
    printf("}\n");
    return 0;
}
