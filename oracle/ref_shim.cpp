/*
 * oracle/ref_shim.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * Thin extern "C" wrapper around the UNMODIFIED reference CPU path (the headers
 * under /root/reference/include and src/autodiff/autodiff.cpp, compiled where
 * they lie -- nothing is copied).  It is built by oracle/Makefile into
 * oracle/_ref/libenoki_ref.so (-ffp-contract=off, parity) and
 * oracle/_ref/libenoki_ref_fast.so (-ffp-contract=fast, the reference's own
 * flags, used only for CPU-baseline timing).
 *
 * Used to (1) pin the C restatement in enoki_oracle.c, (2) generate the golden
 * vectors under tests/golden/, (3) serve as bench.py's `--impl reference` arm.
 * Only tests/, bench.py's cpu_baseline leg and __graft_entry__.smoke() may load
 * it; the product (enoki_b200/) never does.
 *
 * Reference entry points exercised here:
 *   DynamicArray<Packet<float,8>> operators   include/enoki/dynamic.h:275-443
 *   sin/cos/exp/log/...                       include/enoki/array_math.h
 *   PCG32                                     include/enoki/random.h:40-119
 *   erfinv                                    include/enoki/special.h:222-246
 *   gather/scatter_add                        include/enoki/dynamic.h:478-534
 *   hsum/hprod/hmin/hmax/count/any/all        include/enoki/dynamic.h:632-752
 *   Tape<T>::append/backward                  src/autodiff/autodiff.cpp:266-338,838-910
 */
#include <cstdint>
#include <cstring>
#include <cstdio>
#include <cmath>
#include <string>
#include <vector>
#include <memory>
#include <set>
#include <map>
#include <unordered_map>
#include <iostream>
#include <sstream>
#include <algorithm>
#include <stdexcept>
#include <chrono>
#include <thread>

#include <enoki/array.h>
#include <enoki/dynamic.h>
#include <enoki/random.h>
#include <enoki/special.h>
#include <enoki/morton.h>

/* Tape<T>::append()/backward() are private (friend DiffArray); the shim drives
   the tape directly so that test graphs have an exactly known node/edge shape. */
#define private public
#include <enoki/autodiff.h>
#undef private

using namespace enoki;

using FloatP  = Packet<float, 8>;
using FloatX  = DynamicArray<FloatP>;
using UInt32P = Packet<uint32_t, 8>;
using UInt32X = DynamicArray<UInt32P>;
using Int32X  = DynamicArray<Packet<int32_t, 8>>;
using UInt64X = DynamicArray<Packet<uint64_t, 8>>;
using MaskX   = mask_t<FloatX>;
using TapeX   = Tape<FloatX>;

static FloatX  copy_f(const float *p, size_t n)    { return FloatX::copy(p, n); }
static UInt32X copy_u(const uint32_t *p, size_t n) { return UInt32X::copy(p, n); }
static void out_f(const FloatX &v, float *dst, size_t n) {
    if (v.size() == 1 && n > 1) { for (size_t i = 0; i < n; ++i) dst[i] = v.coeff(0); }
    else memcpy(dst, v.data(), n * sizeof(float));
}

extern "C" {

const char *ref_info() {
    static std::string s;
    s = "enoki reference CPU path, Packet<float," + std::to_string(FloatP::Size) + "> "
#if defined(ENOKI_X86_AVX2)
        "AVX2"
#endif
#if defined(ENOKI_X86_FMA)
        "+FMA"
#endif
#if defined(REF_CONTRACT_FAST)
        " (fp-contract=fast)"
#else
        " (fp-contract=off)"
#endif
        ;
    return s.c_str();
}

/* ---- vertical math: unary/binary/ternary on float arrays ---- */
int ref_unary_f32(const char *name, const float *in, float *out, size_t n) {
    FloatX x = copy_f(in, n), r;
    std::string s(name);
    if      (s == "sin")   r = sin(x);
    else if (s == "cos")   r = cos(x);
    else if (s == "tan")   r = tan(x);
    else if (s == "exp")   r = exp(x);
    else if (s == "log")   r = log(x);
    else if (s == "sqrt")  r = sqrt(x);
    else if (s == "rcp")   r = rcp(x);
    else if (s == "rsqrt") r = rsqrt(x);
    else if (s == "abs")   r = abs(x);
    else if (s == "neg")   r = -x;
    else if (s == "floor") r = floor(x);
    else if (s == "ceil")  r = ceil(x);
    else if (s == "round") r = round(x);
    else if (s == "trunc") r = trunc(x);
    else if (s == "asin")  r = asin(x);
    else if (s == "acos")  r = acos(x);
    else if (s == "atan")  r = atan(x);
    else if (s == "sinh")  r = sinh(x);
    else if (s == "cosh")  r = cosh(x);
    else if (s == "tanh")  r = tanh(x);
    else if (s == "cbrt")  r = cbrt(x);
    else if (s == "erfinv") r = erfinv(x);
    else if (s == "erf")   r = erf(x);
    else if (s == "sincos_s") r = sincos(x).first;
    else if (s == "sincos_c") r = sincos(x).second;
    else return -1;
    out_f(r, out, n);
    return 0;
}

int ref_binary_f32(const char *name, const float *a_, const float *b_, float *out, size_t n) {
    FloatX a = copy_f(a_, n), b = copy_f(b_, n), r;
    std::string s(name);
    if      (s == "add")   r = a + b;
    else if (s == "sub")   r = a - b;
    else if (s == "mul")   r = a * b;
    else if (s == "div")   r = a / b;
    else if (s == "min")   r = min(a, b);
    else if (s == "max")   r = max(a, b);
    else if (s == "atan2") r = atan2(a, b);
    else if (s == "pow")   r = pow(a, b);
    else return -1;
    out_f(r, out, n);
    return 0;
}

int ref_fmadd_f32(const float *a_, const float *b_, const float *c_, float *out, size_t n) {
    FloatX a = copy_f(a_, n), b = copy_f(b_, n), c = copy_f(c_, n);
    FloatX r = fmadd(a, b, c);
    out_f(r, out, n);
    return 0;
}

int ref_unary_f64(const char *name, const double *in, double *out, size_t n) {
    using DoubleX = DynamicArray<Packet<double, 4>>;
    DoubleX x = DoubleX::copy(in, n), r;
    std::string s(name);
    if      (s == "sin")  r = sin(x);
    else if (s == "cos")  r = cos(x);
    else if (s == "exp")  r = exp(x);
    else if (s == "log")  r = log(x);
    else if (s == "sqrt") r = sqrt(x);
    else return -1;
    memcpy(out, r.data(), n * sizeof(double));
    return 0;
}

/* float -> int32 conversions used by index math */
void ref_f2i(const float *in, int32_t *out, size_t n) {
    FloatX x = copy_f(in, n);
    Int32X r(x);
    memcpy(out, r.data(), n * 4);
}
void ref_f2u(const float *in, uint32_t *out, size_t n) {
    FloatX x = copy_f(in, n);
    UInt32X r(x);
    memcpy(out, r.data(), n * 4);
}

/* ---- conversions between any two numeric types: DynamicArray<Packet<S, 8>> -> DynamicArray<Packet<D, 8>> through the
        converting constructor (mode 0), floor2int<D> (1) or ceil2int<D> (2); type codes are the ek_type values ---- */
} /* extern "C" */
template <typename S, typename D> static int ref_convert_typed(int mode, const void *in, void *out, size_t n) {
    using SX = DynamicArray<Packet<S, 8>>;
    using DX = DynamicArray<Packet<D, 8>>;
    SX x = SX::copy(in, n);
    DX r;
    if (mode == 0) r = DX(x);
    else if constexpr (std::is_floating_point_v<S> && !std::is_floating_point_v<D>)
        r = mode == 1 ? floor2int<DX>(x) : ceil2int<DX>(x);
    else return -1;
    memcpy(out, r.data(), n * sizeof(D));
    return 0;
}

template <typename S> static int ref_convert_from(int dst, int mode, const void *in, void *out, size_t n) {
    switch (dst) {
        case 1:  return ref_convert_typed<S, int8_t>(mode, in, out, n);
        case 2:  return ref_convert_typed<S, uint8_t>(mode, in, out, n);
        case 3:  return ref_convert_typed<S, int16_t>(mode, in, out, n);
        case 4:  return ref_convert_typed<S, uint16_t>(mode, in, out, n);
        case 5:  return ref_convert_typed<S, int32_t>(mode, in, out, n);
        case 6:  return ref_convert_typed<S, uint32_t>(mode, in, out, n);
        case 7:  return ref_convert_typed<S, int64_t>(mode, in, out, n);
        case 8:  return ref_convert_typed<S, uint64_t>(mode, in, out, n);
        case 10: return ref_convert_typed<S, float>(mode, in, out, n);
        case 11: return ref_convert_typed<S, double>(mode, in, out, n);
        default: return -1;
    }
}
extern "C" {

int ref_convert(int src, int dst, int mode, const void *in, void *out, size_t n) {
    switch (src) {
        case 1:  return ref_convert_from<int8_t>(dst, mode, in, out, n);
        case 2:  return ref_convert_from<uint8_t>(dst, mode, in, out, n);
        case 3:  return ref_convert_from<int16_t>(dst, mode, in, out, n);
        case 4:  return ref_convert_from<uint16_t>(dst, mode, in, out, n);
        case 5:  return ref_convert_from<int32_t>(dst, mode, in, out, n);
        case 6:  return ref_convert_from<uint32_t>(dst, mode, in, out, n);
        case 7:  return ref_convert_from<int64_t>(dst, mode, in, out, n);
        case 8:  return ref_convert_from<uint64_t>(dst, mode, in, out, n);
        case 10: return ref_convert_from<float>(dst, mode, in, out, n);
        case 11: return ref_convert_from<double>(dst, mode, in, out, n);
        default: return -1;
    }
}

/* ---- C1 (tests/dynamic.cpp path): r = a*b + sin(c), operator form ---- */
void ref_c1(const float *a_, const float *b_, const float *c_, float *out, size_t n) {
    FloatX a = copy_f(a_, n), b = copy_f(b_, n), c = copy_f(c_, n);
    FloatX r = a * b + sin(c);
    out_f(r, out, n);
}

/* ---- C2 (SURVEY 8d): fused arith + exp/sin chain, 12 arithmetic nodes ---- */
static FloatX c2_expr(const FloatX &x0, const FloatX &x1, const FloatX &x2, const FloatX &x3) {
    FloatX t = fmadd(x0, x1, x2);
    FloatX u = exp(-(t * t));
    FloatX v = sin(fmadd(x3, u, x0));
    return fmadd(v, x1, sqrt(abs(t)));
}
void ref_c2(const float *x0_, const float *x1_, const float *x2_, const float *x3_,
            float *out, size_t n) {
    FloatX x0 = copy_f(x0_, n), x1 = copy_f(x1_, n), x2 = copy_f(x2_, n), x3 = copy_f(x3_, n);
    FloatX r = c2_expr(x0, x1, x2, x3);
    out_f(r, out, n);
}
/* same, inputs mapped (no copy) and output discarded: used for timing */
double ref_c2_time(float *x0_, float *x1_, float *x2_, float *x3_, size_t n, int reps) {
    FloatX x0 = FloatX::map(x0_, n), x1 = FloatX::map(x1_, n),
           x2 = FloatX::map(x2_, n), x3 = FloatX::map(x3_, n);
    double best = 1e30;
    float sink = 0;
    for (int i = 0; i < reps; ++i) {
        auto t0 = std::chrono::high_resolution_clock::now();
        FloatX r = c2_expr(x0, x1, x2, x3);
        auto t1 = std::chrono::high_resolution_clock::now();
        sink += r.coeff(0);
        best = std::min(best, std::chrono::duration<double>(t1 - t0).count());
    }
    if (sink == 12345.678f) printf(" ");
    return best;
}
/* fused (vectorize()) form of C2: the reference's own best CPU variant (dynamic.h:1025-1074) */
double ref_c2_time_vectorized(float *x0_, float *x1_, float *x2_, float *x3_, float *out_, size_t n, int reps) {
    FloatX x0 = FloatX::map(x0_, n), x1 = FloatX::map(x1_, n),
           x2 = FloatX::map(x2_, n), x3 = FloatX::map(x3_, n), r = FloatX::map(out_, n);
    double best = 1e30;
    for (int i = 0; i < reps; ++i) {
        auto t0 = std::chrono::high_resolution_clock::now();
        vectorize([](auto &&r, auto &&a, auto &&b, auto &&c, auto &&d) {
            using V = std::decay_t<decltype(a)>;
            V t = fmadd(a, b, c);
            V u = exp(-(t * t));
            V v = sin(fmadd(d, u, a));
            r = fmadd(v, b, sqrt(abs(t)));
        }, r, x0, x1, x2, x3);
        auto t1 = std::chrono::high_resolution_clock::now();
        best = std::min(best, std::chrono::duration<double>(t1 - t0).count());
    }
    return best;
}

/* ---- C1 (BASELINE.json configs[0], SURVEY 8d): r = a*b + sin(c) on DynamicArray<Packet<float,8>>, N = 2^20,
        a = linspace(0,1), b = linspace(1,2), c = linspace(-3,3) -- operator form (one heap pass per operator,
        dynamic.h:275-443) and the fused vectorize() form (dynamic.h:1025-1074, tests/dynamic.cpp:192-225).
        Returns the best pass in seconds; out[0] receives r[n/2] so that nothing is optimised away. */
double ref_c1_time_operator(size_t n, int reps, float *out) {
    FloatX a = linspace<FloatX>(0.f, 1.f, n), b = linspace<FloatX>(1.f, 2.f, n), c = linspace<FloatX>(-3.f, 3.f, n);
    double best = 1e30;
    for (int i = 0; i < reps; ++i) {
        auto t0 = std::chrono::high_resolution_clock::now();
        FloatX r = a * b + sin(c);
        auto t1 = std::chrono::high_resolution_clock::now();
        out[0] = r.coeff(n / 2);
        best = std::min(best, std::chrono::duration<double>(t1 - t0).count());
    }
    return best;
}
double ref_c1_time_vectorized(size_t n, int reps, float *out) {
    FloatX a = linspace<FloatX>(0.f, 1.f, n), b = linspace<FloatX>(1.f, 2.f, n), c = linspace<FloatX>(-3.f, 3.f, n);
    FloatX r = zero<FloatX>(n);
    double best = 1e30;
    for (int i = 0; i < reps; ++i) {
        auto t0 = std::chrono::high_resolution_clock::now();
        vectorize([](auto &&r, auto &&a, auto &&b, auto &&c) { r = a * b + sin(c); }, r, a, b, c);
        auto t1 = std::chrono::high_resolution_clock::now();
        out[0] = r.coeff(n / 2);
        best = std::min(best, std::chrono::duration<double>(t1 - t0).count());
    }
    return best;
}

/* ---- PCG32 (random.h:40-119): stream = element index, default state ---- */
void ref_pcg32_u32(uint64_t first, size_t n, size_t draws, uint32_t *out) {
    /* out[d * n + i] = d-th draw of the generator with stream (first + i) */
    using RNG = PCG32<UInt32P>;
    for (size_t i = 0; i < n; i += 8) {
        RNG rng(PCG32_DEFAULT_STATE, arange<RNG::UInt64>() + uint64_t(first + i));
        for (size_t d = 0; d < draws; ++d) {
            UInt32P v = rng.next_uint32();
            for (size_t k = 0; k < 8 && i + k < n; ++k)
                out[d * n + i + k] = v.coeff(k);
        }
    }
}
void ref_pcg32_f32(uint64_t first, size_t n, size_t draws, float *out) {
    using RNG = PCG32<UInt32P>;
    for (size_t i = 0; i < n; i += 8) {
        RNG rng(PCG32_DEFAULT_STATE, arange<RNG::UInt64>() + uint64_t(first + i));
        for (size_t d = 0; d < draws; ++d) {
            auto v = rng.next_float32();
            for (size_t k = 0; k < 8 && i + k < n; ++k)
                out[d * n + i + k] = v.coeff(k);
        }
    }
}

/* ---- C3 (tests/histogram.cpp:41-57) ---- */
/* y = sqrt(2) * erfinv(2u - 1) */
void ref_hist_samples(const float *u_, float *y_, size_t n) {
    FloatX u = copy_f(u_, n);
    FloatX y = float(M_SQRT2) * erfinv(2.f * u - 1.f);
    out_f(y, y_, n);
}
/* idx = UInt32((y+4)*31/8); mask = idx<31; w = gather(table); scatter_add bins(+1), hist(+w) */
void ref_c3(const float *y_, size_t n, const float *table31, uint32_t *idx_out,
            uint32_t *bins, float *hist) {
    const float min_value = -4, max_value = 4;
    const uint32_t bin_count = 31;
    FloatX y = copy_f(y_, n);
    UInt32X idx((y - min_value) * float(bin_count) / (max_value - min_value));
    auto mask = idx >= zero<UInt32X>() && idx < bin_count;
    if (idx_out) memcpy(idx_out, idx.data(), n * 4);
    FloatX w = gather<FloatX>(table31, idx, mask);
    scatter_add(bins, full<UInt32X>(1u, n), idx, mask);
    scatter_add(hist, w, idx, mask);
}
double ref_c3_time(float *y_, size_t n, const float *table31, uint32_t *bins, float *hist, int reps) {
    const float min_value = -4, max_value = 4;
    const uint32_t bin_count = 31;
    FloatX y = FloatX::map(y_, n);
    double best = 1e30;
    for (int i = 0; i < reps; ++i) {
        auto t0 = std::chrono::high_resolution_clock::now();
        UInt32X idx((y - min_value) * float(bin_count) / (max_value - min_value));
        auto mask = idx >= zero<UInt32X>() && idx < bin_count;
        FloatX w = gather<FloatX>(table31, idx, mask);
        scatter_add(bins, full<UInt32X>(1u, n), idx, mask);
        scatter_add(hist, w, idx, mask);
        auto t1 = std::chrono::high_resolution_clock::now();
        best = std::min(best, std::chrono::duration<double>(t1 - t0).count());
    }
    return best;
}

/* ---- gather / scatter / scatter_add on plain arrays (memory.cpp shapes) ---- */
void ref_gather_f32(const float *src, const uint32_t *idx_, const uint8_t *mask_, float *out, size_t n) {
    UInt32X idx = copy_u(idx_, n);
    MaskX mask = neq(DynamicArray<Packet<uint32_t, 8>>(
        UInt32X(DynamicArray<Packet<uint8_t, 8>>::copy(mask_, n))), 0u);
    FloatX r = gather<FloatX>(src, idx, mask);
    out_f(r, out, n);
}
void ref_scatter_add_f32(float *dst, const float *val_, const uint32_t *idx_, const uint8_t *mask_, size_t n) {
    UInt32X idx = copy_u(idx_, n);
    FloatX val = copy_f(val_, n);
    MaskX mask = neq(UInt32X(DynamicArray<Packet<uint8_t, 8>>::copy(mask_, n)), 0u);
    scatter_add(dst, val, idx, mask);
}
void ref_scatter_f32(float *dst, const float *val_, const uint32_t *idx_, const uint8_t *mask_, size_t n) {
    UInt32X idx = copy_u(idx_, n);
    FloatX val = copy_f(val_, n);
    MaskX mask = neq(UInt32X(DynamicArray<Packet<uint8_t, 8>>::copy(mask_, n)), 0u);
    scatter(dst, val, idx, mask);
}

/* ---- horizontal ops (dynamic.h:632-752) ---- */
float ref_hsum_f32(const float *p, size_t n)  { return hsum(copy_f(p, n)); }
float ref_hprod_f32(const float *p, size_t n) { return hprod(copy_f(p, n)); }
float ref_hmin_f32(const float *p, size_t n)  { return hmin(copy_f(p, n)); }
float ref_hmax_f32(const float *p, size_t n)  { return hmax(copy_f(p, n)); }
uint32_t ref_hsum_u32(const uint32_t *p, size_t n) { return hsum(copy_u(p, n)); }
void ref_psum_f32(const float *p, float *out, size_t n) { out_f(psum(copy_f(p, n)), out, n); }
void ref_psum_u32(const uint32_t *p, uint32_t *out, size_t n) {
    UInt32X r = psum(copy_u(p, n)); memcpy(out, r.data(), n * 4);
}

/* ---- Morton codes (morton.h:27-155) ---- */
void ref_morton2_encode(const uint32_t *x_, const uint32_t *y_, uint32_t *out, size_t n) {
    for (size_t i = 0; i < n; ++i)
        out[i] = morton_encode(Array<uint32_t, 2>(x_[i], y_[i]));
}
void ref_morton2_decode(const uint32_t *m, uint32_t *x_, uint32_t *y_, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        auto v = morton_decode<Array<uint32_t, 2>>(m[i]);
        x_[i] = v.x(); y_[i] = v.y();
    }
}

/* ---- safe_mul / safe_fmadd (autodiff.cpp:1191-1221), DynamicArray branch ---- */
/* declared in autodiff.cpp's namespace; re-stated through the tape below.   */

/* ---- Tape (src/autodiff/autodiff.cpp) ---------------------------------- */
/* Generic layered tape used by C4 (SURVEY 8d) and the parity tests:
 *   n_nodes nodes; node i has size node_size[i]; nodes with no in-edges are
 *   leaves.  Edge e: src[e] -> dst[e] with weight array weights + woff[e]
 *   of length wsize[e] (1 or node size).  Edges must be listed grouped by
 *   dst in ascending dst order (tape creation order).  backward() (or
 *   forward()) from `root` (1-based position in node list), seeds grad 1,
 *   and copies the gradient of every node listed in want[] into grads_out
 *   (concatenated; an empty gradient reads as zeros).
 */
static int ref_tape_sweep(bool forward, uint32_t n_nodes, const uint32_t *node_size,
                          uint32_t n_edges, const uint32_t *src, const uint32_t *dst,
                          const float *weights, const uint64_t *woff, const uint32_t *wsize,
                          uint32_t root, uint32_t n_want, const uint32_t *want,
                          float *grads_out, int free_graph) {
    try {
        TapeX *tape = TapeX::get();
        tape->set_graph_simplification(false);
        std::vector<uint32_t> ids(n_nodes + 1, 0);
        uint32_t e = 0;
        for (uint32_t i = 1; i <= n_nodes; ++i) {
            if (e < n_edges && dst[e] == i) {
                ids[i] = tape->append_node(node_size[i - 1], "n");
                while (e < n_edges && dst[e] == i) {
                    /* size-1 operands broadcast their whole first packet (dynamic.h:302-318): fill every lane */
                    FloatX w = wsize[e] == 1 ? full<FloatX>(weights[woff[e]], 1) : FloatX::copy(weights + woff[e], wsize[e]);
                    tape->append_edge(ids[src[e]], ids[i], w);
                    ++e;
                }
            } else {
                ids[i] = tape->append_leaf(node_size[i - 1]);
            }
        }
        if (e != n_edges) return -2;
        if (forward) tape->forward(ids[root], free_graph != 0);
        else tape->backward(ids[root], free_graph != 0);
        size_t off = 0;
        for (uint32_t k = 0; k < n_want; ++k) {
            const FloatX &g = tape->gradient(ids[want[k]]);
            size_t sz = node_size[want[k] - 1];
            if (g.size() == sz) memcpy(grads_out + off, g.data(), sz * 4);
            else if (g.size() == 1) for (size_t j = 0; j < sz; ++j) grads_out[off + j] = g.coeff(0);
            else if (g.size() == 0) for (size_t j = 0; j < sz; ++j) grads_out[off + j] = 0.f;
            else return -3;
            off += sz;
        }
        for (uint32_t i = 1; i <= n_nodes; ++i)
            tape->dec_ref_ext(ids[i]);
        return 0;
    } catch (const std::exception &ex) {
        fprintf(stderr, "ref_tape_%s: %s\n", forward ? "forward" : "backward", ex.what());
        return -1;
    }
}

int ref_tape_backward(uint32_t n_nodes, const uint32_t *node_size,
                      uint32_t n_edges, const uint32_t *src, const uint32_t *dst,
                      const float *weights, const uint64_t *woff, const uint32_t *wsize,
                      uint32_t root, uint32_t n_want, const uint32_t *want,
                      float *grads_out, int free_graph) {
    return ref_tape_sweep(false, n_nodes, node_size, n_edges, src, dst, weights, woff, wsize,
                          root, n_want, want, grads_out, free_graph);
}

int ref_tape_forward(uint32_t n_nodes, const uint32_t *node_size,
                     uint32_t n_edges, const uint32_t *src, const uint32_t *dst,
                     const float *weights, const uint64_t *woff, const uint32_t *wsize,
                     uint32_t root, uint32_t n_want, const uint32_t *want,
                     float *grads_out, int free_graph) {
    return ref_tape_sweep(true, n_nodes, node_size, n_edges, src, dst, weights, woff, wsize,
                          root, n_want, want, grads_out, free_graph);
}

/* Public-API autodiff checks (tests/autodiff.cpp shapes): d/dx of a small expression */
using FloatD = DiffArray<FloatX>;
int ref_ad_expr(int which, const float *x_, size_t n, float *val_out, float *grad_out) {
    try {
        FloatD x = FloatD(FloatX::copy(x_, n));
        set_requires_gradient(x);
        FloatD y;
        switch (which) {
            case 0: y = x * x; break;
            case 1: y = sin(x) * exp(x); break;
            case 2: y = sqrt(abs(x) + 1.f) / (x * x + 2.f); break;
            case 3: y = log(x * x + 1.f) + cos(x); break;
            case 4: y = fmadd(x, x, x) * rcp(x * x + 1.f); break;
            default: return -1;
        }
        FloatD loss = hsum(y);
        out_f(detach(y), val_out, n);
        backward(loss);
        out_f(gradient(x), grad_out, n);
        return 0;
    } catch (const std::exception &ex) {
        fprintf(stderr, "ref_ad_expr: %s\n", ex.what());
        return -1;
    }
}

} /* extern "C" */
