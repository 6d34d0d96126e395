/* Records one pass of the duplication loop and the epilogue of each single precision Carlson integral (carlson_rf,
   carlson_rd, carlson_rc) on CUDAArray<float> arrays mapped over fake device addresses, one primitive node per
   operation, and prints their dry runs as one JSON object.  Nothing is launched.

   The operation sequence is the one ek_math.cuh and tests/ell_oracle.c state for each integral, written here with the
   backend's own primitives (sqrt, rcp, fmadd, max, abs, select, division) one statement per operation, in the order and
   with the operands the templates of special.h record them on this backend; tests/cpp/ell_check.cpp compares the native
   operations with those templates themselves on the device.  A dry run cannot evaluate the loop's none(active), so each
   integral is two programs: one pass (arguments and the active mask in; updated arguments, XYZ and mu_inv -- s and
   inv_mu for R_C -- and the new mask out; R_D also carries sum and num) and the epilogue.  The Python driver
   (tests/test_cpu_elliptic.py) runs the pass until no element is active or ten passes have run, then the epilogue.

   {name: {"in": {role: variable}, "out": {role: variable}, "plan": ek_debug_plan(), "program": ek_debug_program()}}
   with names rf_pass, rf_tail, rd_pass, rd_tail, rc_pass, rc_tail.  Built and run by tests/golden/make_golden_ell.py,
   which stores the output as tests/golden/ell_traced.json. */
#include <enoki/cuda.h>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <utility>
#include <vector>

using namespace enoki;
using FloatC = CUDAArray<float>;
using MaskC = mask_t<FloatC>;
extern "C" char *ek_debug_plan(void);
extern "C" char *ek_debug_program(void);

using Roles = std::vector<std::pair<const char *, uint32_t>>;

static std::string quoted(const char *s) {
    std::string r = "\"";
    for (; *s; ++s) {
        if (*s == '"' || *s == '\\') { r += '\\'; r += *s; }
        else if (*s == '\n') r += "\\n";
        else r += *s;
    }
    return r + "\"";
}

static void roles(const Roles &rs) {
    printf("{");
    for (size_t i = 0; i < rs.size(); ++i) printf("%s\"%s\": %u", i ? ", " : "", rs[i].first, rs[i].second);
    printf("}");
}

static void dump(bool first, const char *name, const Roles &in, const Roles &out) {
    char *plan = ek_debug_plan(), *prog = ek_debug_program();
    if (!plan || !prog) { fprintf(stderr, "%s: dry run failed\n", name); exit(1); }
    printf("%s\"%s\": {\"in\": ", first ? "" : ",\n", name);
    roles(in);
    printf(", \"out\": ");
    roles(out);
    printf(", \"plan\": %s, \"program\": %s}", quoted(plan).c_str(), prog);
    free(plan); free(prog);
}

static uint64_t next_address = 0x7f0001000000ull;
static const size_t n = 1 << 20;
static FloatC input() { FloatC r = FloatC::map((void *) next_address, n); next_address += 0x1000000ull; return r; }
static MaskC mask_input() { MaskC r = MaskC::map((void *) next_address, n); next_address += 0x1000000ull; return r; }

/* ---- R_F and R_D: one pass ---- */
struct Pass3 { FloatC x, y, z, X, Y, Z, mu_inv, sum, num; MaskC active; };

static Pass3 pass3(bool rd, FloatC x, FloatC y, FloatC z, FloatC sum, FloatC num, MaskC active) {
    /* square roots, and lambda = sy*sx + sz*sy + sx*sz as a product followed by two fmas */
    FloatC sx = sqrt(x), sy = sqrt(y), sz = sqrt(z);
    FloatC lambda = sy * sx;
    lambda = fmadd(sz, sy, lambda);
    lambda = fmadd(sx, sz, lambda);
    /* mu: the plain mean (R_F) or the weighted one with weights 1/5, 1/5, 3/5 (R_D), summed left to right */
    FloatC mu;
    if (rd) {
        mu = x * float(1.0 / 5.0);
        mu = mu + y * float(1.0 / 5.0);
        mu = mu + z * float(3.0 / 5.0);
    } else {
        mu = x + y;
        mu = mu + z;
        mu = mu * float(1.0 / 3.0);
    }
    FloatC mu_inv = rcp(mu);
    /* X = 1 - x / mu as one fma of the negated argument */
    FloatC X = fmadd(-x, mu_inv, FloatC(1.f)), Y = fmadd(-y, mu_inv, FloatC(1.f)), Z = fmadd(-z, mu_inv, FloatC(1.f));
    /* eps: the largest magnitude, folded left with max */
    FloatC eps = max(abs(X), abs(Y));
    eps = max(eps, abs(Z));
    active = active & (eps > float(rd ? 0.070154 * 0.6 : 0.070154));
    if (rd) {
        FloatC term = num / (sqrt(z) * (z + lambda));
        sum = select(active, sum + term, sum);
        num = select(active, num * 0.25f, num);
    }
    x = select(active, (x + lambda) * 0.25f, x);
    y = select(active, (y + lambda) * 0.25f, y);
    z = select(active, (z + lambda) * 0.25f, z);
    return { x, y, z, X, Y, Z, mu_inv, sum, num, active };
}

/* ---- R_F: the epilogue, a polynomial in e2 = XY - Z^2 and e3 = XYZ ---- */
static FloatC rf_tail(const FloatC &X, const FloatC &Y, const FloatC &Z, const FloatC &mu_inv) {
    FloatC xy = X * Y;
    FloatC e2 = xy - Z * Z;
    FloatC e3 = xy * Z;
    FloatC t = float(1.0 / 24.0) * e2;
    t = t - float(1.0 / 10.0);
    t = t - float(3.0 / 44.0) * e3;
    t = t * e2;
    FloatC er = t + float(1.0 / 14.0) * e3;
    return sqrt(mu_inv) * (1.f + er);
}

/* ---- R_D: the epilogue ---- */
static FloatC rd_tail(const FloatC &X, const FloatC &Y, const FloatC &Z, const FloatC &mu_inv, const FloatC &sum,
                      const FloatC &num) {
    FloatC ea = X * Y, eb = Z * Z, ec = ea - eb;
    FloatC ed = fmadd(FloatC(-6.f), eb, ea);
    FloatC ee = fmadd(ec, FloatC(2.f), ed);
    /* first part: ed * ((-3/14 + 9/88 ed) - (Z / 4) ee) */
    FloatC a = -float(3.0 / 14.0) + float(9.0 / 88.0) * ed;
    a = a - (0.25f * Z) * ee;
    a = ed * a;
    /* second part: Z * (ee / 6 + Z * (-9/22 ec + (Z * 3/26) ea)) */
    FloatC b = -float(9.0 / 22.0) * ec + (Z * float(3.0 / 26.0)) * ea;
    b = float(1.0 / 6.0) * ee + Z * b;
    b = Z * b;
    FloatC p = a + b;
    FloatC scale = (num * mu_inv) * sqrt(mu_inv);
    return 3.f * sum + scale * (1.f + p);
}

/* ---- R_C: one pass ---- */
struct PassC { FloatC x, y, inv_mu, s; MaskC active; };

static PassC pass_c(FloatC x, FloatC y, MaskC active) {
    FloatC lambda = sqrt(x) * sqrt(y);
    FloatC twice = lambda + y;                       /* lambda + (lambda + y): two roundings */
    lambda = lambda + twice;
    FloatC mu = fmadd(x, FloatC(float(1.0 / 3.0)), y * float(2.0 / 3.0));
    FloatC inv_mu = rcp(mu);
    FloatC s = (y - mu) * inv_mu;
    active = active & (abs(s) > float(0.070154 * 0.48));
    x = select(active, (x + lambda) * 0.25f, x);
    y = select(active, (y + lambda) * 0.25f, y);
    return { x, y, inv_mu, s, active };
}

/* ---- R_C: the epilogue, a polynomial in s evaluated from the innermost term out ---- */
static FloatC rc_tail(const FloatC &s, const FloatC &inv_mu) {
    FloatC q = 0.375f + s * float(9.0 / 22.0);
    q = float(1.0 / 7.0) + s * q;
    q = 0.3f + s * q;
    return sqrt(inv_mu) * (1.f + (s * s) * q);
}

int main() {
    printf("{");
    for (int rd = 0; rd < 2; ++rd) {
        const char *pn = rd ? "rd_pass" : "rf_pass", *tn = rd ? "rd_tail" : "rf_tail";
        {
            FloatC x = input(), y = input(), z = input(), sum = input(), num = input();
            MaskC active = mask_input();
            Pass3 p = pass3(rd, x, y, z, sum, num, active);
            Roles in = { { "x", x.index_() }, { "y", y.index_() }, { "z", z.index_() }, { "active", active.index_() } };
            Roles out = { { "x", p.x.index_() }, { "y", p.y.index_() }, { "z", p.z.index_() },
                          { "X", p.X.index_() }, { "Y", p.Y.index_() }, { "Z", p.Z.index_() },
                          { "mu_inv", p.mu_inv.index_() }, { "active", p.active.index_() } };
            if (rd) {
                in.push_back({ "sum", sum.index_() }); in.push_back({ "num", num.index_() });
                out.push_back({ "sum", p.sum.index_() }); out.push_back({ "num", p.num.index_() });
            }
            dump(rd == 0, pn, in, out);
        }
        {
            FloatC X = input(), Y = input(), Z = input(), mu_inv = input(), sum = input(), num = input();
            FloatC r = rd ? rd_tail(X, Y, Z, mu_inv, sum, num) : rf_tail(X, Y, Z, mu_inv);
            Roles in = { { "X", X.index_() }, { "Y", Y.index_() }, { "Z", Z.index_() }, { "mu_inv", mu_inv.index_() } };
            if (rd) { in.push_back({ "sum", sum.index_() }); in.push_back({ "num", num.index_() }); }
            dump(false, tn, in, { { "r", r.index_() } });
        }
    }
    {
        FloatC x = input(), y = input();
        MaskC active = mask_input();
        PassC p = pass_c(x, y, active);
        dump(false, "rc_pass", { { "x", x.index_() }, { "y", y.index_() }, { "active", active.index_() } },
             { { "x", p.x.index_() }, { "y", p.y.index_() }, { "inv_mu", p.inv_mu.index_() },
               { "s", p.s.index_() }, { "active", p.active.index_() } });
    }
    {
        FloatC s = input(), inv_mu = input();
        FloatC r = rc_tail(s, inv_mu);
        dump(false, "rc_tail", { { "s", s.index_() }, { "inv_mu", inv_mu.index_() } }, { { "r", r.index_() } });
    }
    printf("}\n");
    return 0;
}
