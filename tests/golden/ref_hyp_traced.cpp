/* Records the reference's generic single precision sinh, cosh, tanh, asinh, acosh, atanh, cbrt and sincosh
   (enoki::detail::*_impl of include/enoki/array_math.h) on a CUDAArray<float> mapped over a fake device address, one
   primitive node at a time as they were recorded before these functions had CUDAArray members, and prints the dry run
   of each as one JSON object: {name: {"x": input variable, "out": [result variables], "plan": ek_debug_plan(),
   "program": ek_debug_program()}}.  Nothing is launched.  Built and run by tests/golden/make_golden_hyp.py, which stores
   the output as tests/golden/hyp_traced.json. */
#include <enoki/cuda.h>
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

static void dump(bool first, const char *name, const FloatC &x, const FloatC &a, const FloatC *b) {
    char *plan = ek_debug_plan(), *prog = ek_debug_program();
    if (!plan || !prog) { fprintf(stderr, "%s: dry run failed\n", name); exit(1); }
    printf("%s\"%s\": {\"x\": %u, \"out\": [%u", first ? "" : ",\n", name, x.index_(), a.index_());
    if (b) printf(", %u", b->index_());
    printf("], \"plan\": %s, \"program\": %s}", quoted(plan).c_str(), prog);
    free(plan); free(prog);
}

int main() {
    const size_t n = 1 << 20;
    FloatC x = FloatC::map((void *) 0x7f0001000000ull, n);
    printf("{");
    { FloatC r = detail::sinh_impl(x);  dump(true, "sinh", x, r, nullptr); }
    { FloatC r = detail::cosh_impl(x);  dump(false, "cosh", x, r, nullptr); }
    { FloatC r = detail::tanh_impl(x);  dump(false, "tanh", x, r, nullptr); }
    { FloatC r = detail::asinh_impl(x); dump(false, "asinh", x, r, nullptr); }
    { FloatC r = detail::acosh_impl(x); dump(false, "acosh", x, r, nullptr); }
    { FloatC r = detail::atanh_impl(x); dump(false, "atanh", x, r, nullptr); }
    { FloatC r = detail::cbrt_impl(x);  dump(false, "cbrt", x, r, nullptr); }
    { auto r = detail::sincosh_impl(x); dump(false, "sincosh", x, r.first, &r.second); }
    printf("}\n");
    return 0;
}
