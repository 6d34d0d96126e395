/*
 * ek_sweep_common.cuh -- device helpers shared by the general sweep kernel (ek_sweep.cu) and the 32-bit fast
 * kernel (ek_sweep_fast.cu): shared-memory / mbarrier / TMA wrappers, x86 conversion semantics of the CPU path,
 * the generic reduction combine, warp-aggregated global atomics.
 */
#pragma once
#ifndef EK_HOST_EMU          /* tests/cpu_kernel: the fast kernel compiled as host code, see cuda_shim.h */
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#endif
#include <stdint.h>
#include "ek_isa.h"
#include "ek_math.cuh"

namespace {

#ifdef EK_HOST_EMU
/* host emulation (tests/cpu_kernel): shared-space addresses are offsets into the CTA's buffer, an mbarrier (expected
   arrival count 1) is a word {bit 0: parity of the current phase, bit 1: the phase's arrival has been made, bits 32..:
   pending transaction bytes}, a TMA bulk copy is a memcpy.  A phase completes when it has its arrival AND no pending
   bytes: bytes may be expected before the arrival (an early release), and then the barrier must not flip early. */
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t) __cvta_generic_to_shared(p); }
inline uint8_t *emu_smem_ptr(uint32_t addr) { return emu::smem_ + (addr - emu::SMEM_WINDOW); }
/* atomically apply (arrive?, +add bytes, -sub bytes) and complete the phase when it is due */
inline void emu_mbar_update(uint64_t *bar, bool arrive, uint32_t add, uint32_t sub) {
    uint64_t w = __atomic_load_n(bar, __ATOMIC_SEQ_CST), nw;
    do {
        const uint64_t tx = (w >> 32) + add;
        if (tx < sub) emu::trap("mbarrier transaction count underflow");
        const uint64_t left = tx - sub;
        const bool arrived = ((w >> 1) & 1u) || arrive;
        if (arrive && ((w >> 1) & 1u)) emu::trap("second arrival on a count-1 mbarrier phase");
        nw = (left << 32) | (w & 1u) | (arrived ? 2u : 0u);
        if (arrived && left == 0) nw = (w & 1u) ^ 1u;                 /* phase complete: next parity, no arrival yet */
    } while (!__atomic_compare_exchange_n(bar, &w, nw, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t) { __atomic_store_n(bar, 0ull, __ATOMIC_SEQ_CST); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) { emu_mbar_update(bar, true, bytes, 0); }
__device__ __forceinline__ void mbar_expect_tx_only(uint64_t *bar, uint32_t bytes) { emu_mbar_update(bar, false, bytes, 0); }
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar_addr, uint32_t parity) {
    const uint64_t w = __atomic_load_n(reinterpret_cast<uint64_t *>(emu_smem_ptr(bar_addr)), __ATOMIC_SEQ_CST);
    return ((uint32_t) w & 1u) != parity;
}
__device__ __forceinline__ void mbar_wait_watchdog(uint64_t *bar, uint32_t parity) {
    const uint32_t a = smem_u32(bar);
    for (unsigned long spins = 0; !mbar_try_wait(a, parity); ++spins) { if (spins > 200000000ul) emu::trap("mbarrier never completed"); sched_yield(); }
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) { mbar_wait_watchdog(bar, parity); }
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const void *src, uint32_t bytes, uint64_t *bar) {
    if (((uintptr_t) src & 15u) || (bytes & 15u) || (smem_u32(dst_smem) & 15u)) emu::trap("misaligned bulk copy");
    memcpy(dst_smem, src, bytes);
    emu_mbar_update(bar, false, 0, bytes);
}
__device__ __forceinline__ void tma_prefetch_l2(const void *, uint32_t) {}
__device__ __forceinline__ void fence_barrier_init() {}
__device__ __forceinline__ void fence_proxy_async() {}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    if (addr & 15u) emu::trap("misaligned 128-bit shared load");
    return *reinterpret_cast<const uint4 *>(emu_smem_ptr(addr));
}
__device__ __forceinline__ void sts128(uint32_t addr, uint4 v) {
    if (addr & 15u) emu::trap("misaligned 128-bit shared store");
    *reinterpret_cast<uint4 *>(emu_smem_ptr(addr)) = v;
}
#else
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return (uint32_t) __cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
                 :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
/* add expected transaction bytes without arriving (early partial issue of a tile) */
__device__ __forceinline__ void mbar_expect_tx_only(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
/* the same wait with a watchdog: a barrier that does not complete within ~2 s (a lost transaction count, i.e. a bug)
   traps -- the launch fails with an error instead of hanging the device */
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar_addr, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n" : "=r"(ok) : "r"(bar_addr), "r"(parity) : "memory");
    return ok;
}
__device__ __forceinline__ void mbar_wait_watchdog(uint64_t *bar, uint32_t parity) {
    const uint32_t a = smem_u32(bar);
    if (mbar_try_wait(a, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(a, parity)) {
        if (clock64() - t0 > 4000000000ll) __trap();
    }
}
/* TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP) */
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        :: "r"(smem_u32(dst_smem)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
/* warm the L2 with the tile this CTA will stage next (SASS: UBLKPF) */
__device__ __forceinline__ void tma_prefetch_l2(const void *src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

/* shared-space 128-bit accesses with explicit 32-bit addresses (keeps the interpreter loop free of
   generic->shared address conversions) */
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, uint4 v) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" :: "r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
#endif
/* value the compiler must keep in a register (no rematerialisation, no hoisting across this point) */
__device__ __forceinline__ uint32_t opaque(uint32_t x) { asm volatile("" : "+r"(x)); return x; }

__device__ __forceinline__ uint64_t mk64(uint32_t lo, uint32_t hi) { return ((uint64_t) hi << 32) | lo; }
__device__ __forceinline__ double   mkd(uint32_t lo, uint32_t hi) { return __hiloint2double((int) hi, (int) lo); }
__device__ __forceinline__ uint32_t dlo(double d) { return (uint32_t) __double2loint(d); }
__device__ __forceinline__ uint32_t dhi(double d) { return (uint32_t) __double2hiint(d); }

/* x86 conversion semantics of the CPU path for out-of-range values */
__device__ __forceinline__ int32_t f2i(float x, uint32_t mode) {
    if (!(x >= -2147483648.f && x < 2147483648.f)) return (int32_t) 0x80000000;
    switch (mode) {
        case EK_RM: return __float2int_rd(x);
        case EK_RP: return __float2int_ru(x);
        case EK_RN: return __float2int_rn(x);
        default:    return __float2int_rz(x);
    }
}
__device__ __forceinline__ uint32_t f2u(float x, uint32_t mode) {
    /* AVX2 has no unsigned conversion: the CPU path (array_avx2.h) converts a value r >= 2^31 as
       cvttps2dq(r - 2^31) + 2^31 and anything else as cvttps2dq(r), where r = floor / ceil / trunc (x).  So r in
       [0, 2^32) is exact, r in [-2^31, 0) wraps like int32, NaN and r < -2^31 give 0x80000000, r >= 2^32 gives 0 */
    float r;
    switch (mode) {
        case EK_RM: r = floorf(x); break;
        case EK_RP: r = ceilf(x); break;
        case EK_RN: r = rintf(x); break;
        default:    r = truncf(x); break;
    }
    if (r >= 2147483648.f) return (uint32_t) f2i(r - 2147483648.f, EK_RZ) + 0x80000000u;
    return (uint32_t) f2i(r, EK_RZ);
}
/* cvttpd2dq of the rounded value: the range test follows the rounding (ceil of a double just below 2^31 is out of range) */
__device__ __forceinline__ int32_t d2i(double x, uint32_t mode) {
    double r;
    switch (mode) {
        case EK_RM: r = floor(x); break;
        case EK_RP: r = ceil(x); break;
        case EK_RN: r = rint(x); break;
        default:    r = trunc(x); break;
    }
    if (!(r >= -2147483648.0 && r < 2147483648.0)) return (int32_t) 0x80000000;
    return __double2int_rz(r);
}
__device__ __forceinline__ long long d2ll(double x, uint32_t mode) {
    if (!(x >= -9223372036854775808.0 && x < 9223372036854775808.0)) return (long long) 0x8000000000000000ull;
    switch (mode) {
        case EK_RM: return __double2ll_rd(x);
        case EK_RP: return __double2ll_ru(x);
        case EK_RN: return __double2ll_rn(x);
        default:    return __double2ll_rz(x);
    }
}
__device__ __forceinline__ long long f2ll(float x, uint32_t mode) {
    if (!(x >= -9223372036854775808.f && x < 9223372036854775808.f)) return (long long) 0x8000000000000000ull;
    switch (mode) {
        case EK_RM: return __float2ll_rd(x);
        case EK_RP: return __float2ll_ru(x);
        case EK_RN: return __float2ll_rn(x);
        default:    return __float2ll_rz(x);
    }
}
/* to uint64: [2^63, 2^64) (where every float / double is an integer) is exact, anything else as the int64 conversion */
__device__ __forceinline__ uint64_t f2ull(float x, uint32_t mode) {
    if (x >= 9223372036854775808.f && x < 18446744073709551616.f)
        return (uint64_t) f2ll(x - 9223372036854775808.f, EK_RZ) + 0x8000000000000000ull;
    return (uint64_t) f2ll(x, mode);
}
__device__ __forceinline__ uint64_t d2ull(double x, uint32_t mode) {
    if (x >= 9223372036854775808.0 && x < 18446744073709551616.0)
        return (uint64_t) d2ll(x - 9223372036854775808.0, EK_RZ) + 0x8000000000000000ull;
    return (uint64_t) d2ll(x, mode);
}

/* Float16 is a storage format: a value is its binary16 bit pattern, zero-extended in a 32-bit register.  f32 -> f16
   rounds to nearest even (cvt.rn.f16.f32: |x| >= 65520 gives inf, half subnormals exact, f32 subnormals give 0), the
   reference's float32_to_float16 with F16C; f16 -> f32 is exact (cvt.f32.f16) */
#ifdef EK_HOST_EMU
/* (host build: the same two conversions in integer arithmetic, independent of the host's F16C; NaN gives the canonical
   0x7fff / 0x7fffffff as on the H100) */
inline uint32_t f32_to_f16(float f) {
    uint32_t x; memcpy(&x, &f, 4);
    const uint32_t sign = (x >> 16) & 0x8000u, ax = x & 0x7fffffffu;
    if (ax > 0x7f800000u) return 0x7fffu;
    if (ax >= 0x477ff000u) return sign | 0x7c00u;                                   /* |x| >= 65520: inf */
    if (ax >= 0x38800000u) return sign | ((ax + 0xfffu + ((ax >> 13) & 1u) - 0x38000000u) >> 13);   /* normal half */
    if (ax < 0x33000000u) return sign;                                              /* below 2^-25 (2^-25 ties to 0) */
    const uint32_t shift = 126u - (ax >> 23), m = (ax & 0x7fffffu) | 0x800000u;     /* subnormal: m * 2^-shift units of 2^-24 */
    uint32_t k = m >> shift;
    const uint32_t rem = m & ((1u << shift) - 1u), halfway = 1u << (shift - 1u);
    if (rem > halfway || (rem == halfway && (k & 1u))) ++k;
    return sign | k;
}
inline float f16_to_f32(uint32_t h) {
    const uint32_t sign = (h & 0x8000u) << 16, e = (h >> 10) & 0x1fu, m = h & 0x3ffu;
    uint32_t x;
    if (e == 0x1fu) x = m ? 0x7fffffffu : (sign | 0x7f800000u);
    else if (e) x = sign | ((e + 112u) << 23) | (m << 13);
    else { const float f = (float) m * 0x1p-24f; memcpy(&x, &f, 4); x |= sign; }
    float r; memcpy(&r, &x, 4); return r;
}
#else
__device__ __forceinline__ uint32_t f32_to_f16(float x) { return (uint32_t) __half_as_ushort(__float2half_rn(x)); }
__device__ __forceinline__ float f16_to_f32(uint32_t h) { return __half2float(__ushort_as_half((unsigned short) h)); }
#endif

/* generic 64-bit-carried reduction combine (used by RACC slow path / RFIN) */
__device__ __noinline__ uint64_t red_combine(uint32_t kind, uint32_t cls, uint64_t a, uint64_t b) {
    switch (cls) {
        case EK_RC_F32: {
            float x = __uint_as_float((uint32_t) a), y = __uint_as_float((uint32_t) b), r;
            switch (kind) {
                case EK_RED_SUM:  r = __fadd_rn(x, y); break;
                case EK_RED_PROD: r = __fmul_rn(x, y); break;
                case EK_RED_MIN:  r = ekm::min_x86(y, x); break;
                default:          r = ekm::max_x86(y, x); break;
            }
            return __float_as_uint(r);
        }
        case EK_RC_I32: {
            int32_t x = (int32_t) a, y = (int32_t) b, r;
            switch (kind) {
                case EK_RED_SUM:  r = x + y; break;
                case EK_RED_PROD: r = x * y; break;
                case EK_RED_MIN:  r = min(x, y); break;
                default:          r = max(x, y); break;
            }
            return (uint32_t) r;
        }
        case EK_RC_U32: {
            uint32_t x = (uint32_t) a, y = (uint32_t) b, r;
            switch (kind) {
                case EK_RED_SUM:  r = x + y; break;
                case EK_RED_PROD: r = x * y; break;
                case EK_RED_MIN:  r = min(x, y); break;
                default:          r = max(x, y); break;
            }
            return r;
        }
        case EK_RC_F64: {
            double x = __longlong_as_double((long long) a), y = __longlong_as_double((long long) b), r;
            switch (kind) {
                case EK_RED_SUM:  r = __dadd_rn(x, y); break;
                case EK_RED_PROD: r = __dmul_rn(x, y); break;
                case EK_RED_MIN:  r = ekm::min_x86(y, x); break;
                default:          r = ekm::max_x86(y, x); break;
            }
            return (uint64_t) __double_as_longlong(r);
        }
        case EK_RC_I64: {
            long long x = (long long) a, y = (long long) b, r;
            switch (kind) {
                case EK_RED_SUM:  r = x + y; break;
                case EK_RED_PROD: r = x * y; break;
                case EK_RED_MIN:  r = min(x, y); break;
                default:          r = max(x, y); break;
            }
            return (uint64_t) r;
        }
        default: {
            uint64_t r;
            switch (kind) {
                case EK_RED_SUM:  r = a + b; break;
                case EK_RED_PROD: r = a * b; break;
                case EK_RED_MIN:  r = min(a, b); break;
                default:          r = max(a, b); break;
            }
            return r;
        }
    }
}

__device__ __forceinline__ uint64_t shfl_xor64(uint64_t v, int m) {
    uint32_t lo = __shfl_xor_sync(0xffffffffu, (uint32_t) v, m);
    uint32_t hi = __shfl_xor_sync(0xffffffffu, (uint32_t) (v >> 32), m);
    return mk64(lo, hi);
}

/* warp-aggregated red.global.add: lanes that target the same address are combined with
   shuffles first so that one atomic per distinct address leaves the warp */
template <typename T>
__device__ __forceinline__ void warp_agg_atomic_add(T *addr, T value, bool active) {
    unsigned amask = __ballot_sync(0xffffffffu, active);
    if (!active) return;
    unsigned lane = threadIdx.x & 31u;
    unsigned peers = __match_any_sync(amask, (unsigned long long) addr);
    if (__all_sync(amask, peers == (1u << lane))) {      /* conflict-free warp: fast path */
        atomicAdd(addr, value);
        return;
    }
    unsigned leader = __ffs(peers) - 1;
    unsigned rem = peers & ~(1u << leader);              /* what the leader still has to pull */
    T sum = value;
    /* every lane walks its own peer list; lanes stay converged on the shuffle */
    while (__any_sync(amask, rem != 0)) {
        unsigned src = rem ? (__ffs(rem) - 1) : lane;
        T v = __shfl_sync(amask, value, src);
        if (rem) { sum += v; rem &= rem - 1; }
    }
    if (lane == leader) atomicAdd(addr, sum);
}

/* rarely used, fat double-precision routines are kept out of line so that the interpreter loop stays
   small (instruction-cache footprint of the hot cases) */
__device__ __noinline__ double ek_f64_fn(int which, double x) {
    switch (which) {
        case 0: return ekm::exp_f64(x);
        case 1: return ekm::log_f64(x);
        case 2: return ekm::sin_f64(x);
        default: return ekm::cos_f64(x);
    }
}
/* which: 0 signed div, 1 unsigned div, 2 signed mod, 3 unsigned mod -- x86-style results for /0 are
   not defined by the reference; CUDA semantics with guards against traps */
__device__ __noinline__ long long ek_div64(int which, long long a, long long b) {
    switch (which) {
        case 0: return b == 0 ? 0 : (b == -1 ? (long long) (0ull - (uint64_t) a) : a / b);
        case 1: return (long long) ((uint64_t) b == 0 ? ~0ull : (uint64_t) a / (uint64_t) b);
        case 2: return (b == 0 || b == -1) ? 0 : a % b;
        default: return (long long) ((uint64_t) b == 0 ? (uint64_t) a : (uint64_t) a % (uint64_t) b);
    }
}
__device__ __forceinline__ uint64_t ek_div64(int which, uint64_t a, uint64_t b) {
    return (uint64_t) ek_div64(which, (long long) a, (long long) b);
}

struct Desc {          /* privatised-bins / staged-table descriptor: 4 words in the uniform pool */
    uint32_t smem_off; /* byte offset inside the extra region                         */
    uint32_t count;    /* number of 32-bit entries                                    */
    uint32_t copies;   /* number of per-warp copies (bins) / 1 (tables)               */
    uint32_t ptr_uni;  /* uniform index of the global base pointer                    */
};


} // namespace
