/* Records the reference's generic single precision pow, frexp and hypot (include/enoki/array_math.h) and
   dawson and erfi (include/enoki/special.h) on CUDAArray<float> arrays mapped over fake device addresses, one primitive
   node at a time as they were recorded before these functions were native (detail::pow_impl ... and the templates with
   explicit arguments pick the generic bodies over cuda.h's members and overloads), and prints the dry run of each as
   one JSON object: {name: {"x": input variable, "y": second input variable (binary functions), "out": [result
   variables], "plan": ek_debug_plan(), "program": ek_debug_program()}}.  Nothing is launched.  Built and run by
   tests/golden/make_golden_math.py, which stores the output as tests/golden/math_traced.json. */
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

static void dump(bool first, const char *name, const FloatC &x, const FloatC *y, const FloatC &r, const FloatC *r2) {
    char *plan = ek_debug_plan(), *prog = ek_debug_program();
    if (!plan || !prog) { fprintf(stderr, "%s: dry run failed\n", name); exit(1); }
    printf("%s\"%s\": {\"x\": %u, ", first ? "" : ",\n", name, x.index_());
    if (y) printf("\"y\": %u, ", y->index_());
    printf("\"out\": [%u", r.index_());
    if (r2) printf(", %u", r2->index_());
    printf("], \"plan\": %s, \"program\": %s}", quoted(plan).c_str(), prog);
    free(plan); free(prog);
}

int main() {
    const size_t n = 1 << 20;
    FloatC x = FloatC::map((void *) 0x7f0001000000ull, n), y = FloatC::map((void *) 0x7f0002000000ull, n);
    printf("{");
    { FloatC r = detail::pow_impl<FloatC>(x, y);   dump(true, "pow", x, &y, r, nullptr); }
    { auto r = detail::frexp_impl<FloatC>(x);      dump(false, "frexp", x, nullptr, r.first, &r.second); }
    { FloatC r = hypot<FloatC, FloatC>(x, y);      dump(false, "hypot", x, &y, r, nullptr); }
    { FloatC r = dawson<FloatC>(x);                dump(false, "dawson", x, nullptr, r, nullptr); }
    /* special.h:267-271 erfi<FloatC> calls dawson unqualified, which finds cuda.h's overload: the traced body is this */
    { FloatC r = float(M_2_SQRTPI) * dawson<FloatC>(x) * exp(x * x); dump(false, "erfi", x, nullptr, r, nullptr); }
    printf("}\n");
    return 0;
}
