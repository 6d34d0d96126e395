/*
    enoki/cuda.h (enoki_b200) -- drop-in replacement of the reference's
    include/enoki/cuda.h for the H100-native backend.

    Put this repository's include/ directory BEFORE the reference's on the include path:

        g++ -std=c++17 -I<enoki_b200>/include -I<enoki>/include app.cpp -lenoki_b200

    It provides `enoki::CUDAArray<T>` with the member set the reference's router
    (array_router.h:23-258, array_math.h:110-253, array_struct.h:8-123, array_utils.h:22-47)
    dispatches to -- same names, argument meaning and error behaviour -- but every member records
    an *opcode* through the C ABI of libenoki_b200.so (include/enoki_b200.h) instead of a PTX
    string (reference: include/enoki/cuda.h:205-954).  The free functions of the reference's
    library interface (cuda.h:26-200) are kept as thin inline wrappers so that existing callers
    (`cuda_eval()`, `cuda_sync()`, `cuda_malloc_trim()`, ...) compile unchanged.

    User errors are rethrown as std::runtime_error with the runtime's message, CUDA failures
    terminate the process -- both like the reference (jit.cu:207-212,777-782; common.cu:268-286).
*/
#pragma once

#define ENOKI_CUDA_H 1
#if !defined(ENOKI_CUDA)
#  define ENOKI_CUDA 1
#endif

#include <enoki/array.h>
#include <enoki_b200.h>
#include <enoki_b200_dlpack.h>
#include <stdexcept>
#include <string>
#include <vector>
#include <cstring>

NAMESPACE_BEGIN(enoki)

// -----------------------------------------------------------------------
//! @{ \name Library interface of the reference (cuda.h:26-200) on top of the C ABI
// -----------------------------------------------------------------------

namespace detail {
    [[noreturn]] inline void ek_throw() { throw std::runtime_error(ek_last_error()); }
    inline uint32_t ek_chk(uint32_t h) { if (ENOKI_UNLIKELY(h == 0)) ek_throw(); return h; }
    inline void ek_chk_rc(int rc) { if (ENOKI_UNLIKELY(rc != 0)) ek_throw(); }
    inline uint32_t ek_append(EnokiType t, ek_op op, uint32_t a = 0, uint32_t b = 0, uint32_t c = 0, uint64_t imm = 0) {
        return ek_chk(ek_trace_append((ek_type) t, op, a, b, c, imm));
    }
}

inline void cuda_init() { detail::ek_chk_rc(ek_init()); }
inline void cuda_shutdown() { ek_shutdown(); }
/* (default arguments of cuda_eval / cuda_set_scatter_gather_operand come from the forward declarations in
   the reference's array_router.h:963-967) */
inline void cuda_eval(bool /* log_assembly */) { detail::ek_chk_rc(ek_eval()); }
/* the reference's cuda_printf template (array_router.h:971-975) records through this; see ek_trace_printf() */
inline void cuda_trace_printf(const char *fmt, uint32_t narg, uint32_t *args) { detail::ek_chk_rc(ek_trace_printf(fmt, narg, args)); }
inline void cuda_eval_var(uint32_t index, bool = false) { detail::ek_chk_rc(ek_eval_var(index)); }
inline void cuda_inc_ref_ext(uint32_t i) { ek_inc_ref_ext(i); }
inline void cuda_dec_ref_ext(uint32_t i) { ek_dec_ref_ext(i); }
inline size_t cuda_var_size(uint32_t i) { return ek_var_size(i); }
inline void *cuda_var_ptr(uint32_t i) { return ek_var_ptr(i); }
inline uint32_t cuda_var_set_size(uint32_t i, size_t size, bool copy = false) { return detail::ek_chk(ek_var_set_size(i, size, copy)); }
inline void cuda_var_mark_dirty(uint32_t i) { detail::ek_chk_rc(ek_var_mark_dirty(i)); }
inline void cuda_var_set_label(uint32_t i, const char *l) { ek_var_set_label(i, l); }
inline void cuda_var_mark_side_effect(uint32_t i) { detail::ek_chk_rc(ek_var_mark_side_effect(i)); }
inline void cuda_set_scatter_gather_operand(uint32_t i, bool gather) { detail::ek_chk_rc(ek_set_scatter_gather_operand(i, gather)); }
inline uint32_t cuda_var_copy_to_device(EnokiType t, size_t size, const void *v) { return detail::ek_chk(ek_var_copy_to_device((ek_type) t, size, v)); }
inline uint32_t cuda_var_register_ptr(const void *p) { return detail::ek_chk(ek_var_register_ptr(p)); }
inline uint32_t cuda_var_register(EnokiType t, size_t size, void *p, bool dealloc) { return detail::ek_chk(ek_var_register((ek_type) t, size, p, dealloc)); }
inline void cuda_fetch_element(void *dst, uint32_t i, size_t off, size_t size) { detail::ek_chk_rc(ek_fetch_element(dst, i, off, size)); }
inline void cuda_memcpy_to_device(void *d, const void *s, size_t n) { ek_memcpy_to_device(d, s, n); }
inline void cuda_memcpy_to_device_async(void *d, const void *s, size_t n) { ek_memcpy_to_device_async(d, s, n); }
inline void cuda_memcpy_from_device(void *d, const void *s, size_t n) { ek_memcpy_from_device(d, s, n); }
inline void cuda_memcpy_from_device_async(void *d, const void *s, size_t n) { ek_memcpy_from_device_async(d, s, n); }
inline void cuda_mem_get_info(size_t *f, size_t *t) { ek_mem_get_info(f, t); }
inline void *cuda_malloc(size_t n) { return ek_malloc(n); }
inline void *cuda_managed_malloc(size_t n) { return ek_managed_malloc(n); }
inline void *cuda_host_malloc(size_t n) { return ek_host_malloc(n); }
inline void cuda_fill(uint8_t *p, uint8_t v, size_t n) { ek_fill(p, 1, v, n); }
inline void cuda_fill(uint16_t *p, uint16_t v, size_t n) { ek_fill(p, 2, v, n); }
inline void cuda_fill(uint32_t *p, uint32_t v, size_t n) { ek_fill(p, 4, v, n); }
inline void cuda_fill(uint64_t *p, uint64_t v, size_t n) { ek_fill(p, 8, v, n); }
inline void cuda_reverse(uint8_t *o, const uint8_t *i, size_t n) { ek_reverse(o, i, 1, n); }
inline void cuda_reverse(uint16_t *o, const uint16_t *i, size_t n) { ek_reverse(o, i, 2, n); }
inline void cuda_reverse(uint32_t *o, const uint32_t *i, size_t n) { ek_reverse(o, i, 4, n); }
inline void cuda_reverse(uint64_t *o, const uint64_t *i, size_t n) { ek_reverse(o, i, 8, n); }
inline void cuda_free(void *p) { ek_free(p); }
inline void cuda_host_free(void *p) { ek_host_free(p); }
inline void cuda_malloc_trim() { ek_malloc_trim(); }
inline void cuda_sync() { ek_sync(); }
inline char *cuda_whos() { return ek_whos(); }
inline void cuda_make_managed(uint32_t i) { detail::ek_chk_rc(ek_make_managed(i)); }
inline void cuda_register_callback(void (*cb)(void *), void *p) { ek_register_callback(cb, p); }
inline void cuda_unregister_callback(void (*cb)(void *), void *p) { detail::ek_chk_rc(ek_unregister_callback(cb, p)); }
inline void cuda_set_log_level(uint32_t l) { ek_set_log_level(l); }
inline uint32_t cuda_log_level() { return ek_log_level(); }

template <typename T> T *cuda_psum(size_t n, const T *p) { T *r = (T *) ek_psum((ek_type) enoki_type_v<T>, n, p); if (!r) detail::ek_throw(); return r; }
template <typename T> T *cuda_hsum(size_t n, const T *p) { T *r = (T *) ek_hsum((ek_type) enoki_type_v<T>, n, p); if (!r) detail::ek_throw(); return r; }
template <typename T> T *cuda_hprod(size_t n, const T *p) { T *r = (T *) ek_hprod((ek_type) enoki_type_v<T>, n, p); if (!r) detail::ek_throw(); return r; }
template <typename T> T *cuda_hmax(size_t n, const T *p) { T *r = (T *) ek_hmax((ek_type) enoki_type_v<T>, n, p); if (!r) detail::ek_throw(); return r; }
template <typename T> T *cuda_hmin(size_t n, const T *p) { T *r = (T *) ek_hmin((ek_type) enoki_type_v<T>, n, p); if (!r) detail::ek_throw(); return r; }
inline size_t cuda_count(size_t n, const bool *m) { return ek_count(n, (const uint8_t *) m); }
inline bool cuda_all(size_t n, const bool *m) { return ek_all(n, (const uint8_t *) m) != 0; }
inline bool cuda_any(size_t n, const bool *m) { return ek_any(n, (const uint8_t *) m) != 0; }
template <typename T> void cuda_compress(size_t n, const T *data, const bool *mask, T **out, size_t *out_size) {
    detail::ek_chk_rc(ek_compress((ek_type) enoki_type_v<T>, n, data, (const uint8_t *) mask, (void **) out, out_size));
}
inline void cuda_partition(size_t size, const void **ptrs, void ***unique_out, uint32_t **counts_out, uint32_t ***perm_out) {
    detail::ek_chk_rc(ek_partition(size, ptrs, unique_out, counts_out, perm_out));
}

//! @}
// -----------------------------------------------------------------------

template <typename Value>
struct CUDAArray : ArrayBase<value_t<Value>, CUDAArray<Value>> {
    template <typename T> friend struct CUDAArray;
    using Index = uint32_t;

    static constexpr EnokiType Type = enoki_type_v<Value>;
    static constexpr bool IsCUDA = true;
    template <typename T> using ReplaceValue = CUDAArray<T>;
    using MaskType = CUDAArray<bool>;
    using ArrayType = CUDAArray;

    // ---- handle semantics: intrusive external reference count (cuda.h:216-258) ----
    CUDAArray() = default;
    ~CUDAArray() {
        ek_dec_ref_ext(m_index);
        if constexpr (std::is_pointer_v<Value> || std::is_same_v<Value, uintptr_t>) delete m_cached_partition;
    }
    CUDAArray(const CUDAArray &a) : m_index(a.m_index) { ek_inc_ref_ext(m_index); }
    CUDAArray(CUDAArray &&a) noexcept : m_index(a.m_index) {
        a.m_index = 0;
        if constexpr (std::is_pointer_v<Value> || std::is_same_v<Value, uintptr_t>) {
            m_cached_partition = a.m_cached_partition; a.m_cached_partition = nullptr;
        }
    }
    CUDAArray &operator=(const CUDAArray &a) {
        ek_inc_ref_ext(a.m_index);
        ek_dec_ref_ext(m_index);
        m_index = a.m_index;
        if constexpr (std::is_pointer_v<Value> || std::is_same_v<Value, uintptr_t>) { delete m_cached_partition; m_cached_partition = nullptr; }
        return *this;
    }
    CUDAArray &operator=(CUDAArray &&a) noexcept {
        std::swap(m_index, a.m_index);
        if constexpr (std::is_pointer_v<Value> || std::is_same_v<Value, uintptr_t>) std::swap(m_cached_partition, a.m_cached_partition);
        return *this;
    }

    /// Converting constructor: float -> int truncates, int -> float rounds to nearest (cuda.h:236-247)
    template <typename T> CUDAArray(const CUDAArray<T> &v)
        : m_index(detail::ek_append(Type, EK_OP_CVT, v.index_())) { }

    /// Reinterpreting constructor (cuda.h:249-258)
    template <typename T> CUDAArray(const CUDAArray<T> &v, detail::reinterpret_flag) {
        static_assert(sizeof(T) == sizeof(Value));
        if (std::is_integral_v<T> != std::is_integral_v<Value>) {
            m_index = detail::ek_append(Type, EK_OP_BITCAST, v.index_());
        } else {
            m_index = v.index_();
            ek_inc_ref_ext(m_index);
        }
    }

    template <typename T, enable_if_t<std::is_scalar_v<T>> = 0>
    CUDAArray(const T &value, detail::reinterpret_flag) : CUDAArray(memcpy_cast<Value>(value)) { }

    template <typename T, enable_if_t<std::is_scalar_v<T>> = 0>
    CUDAArray(T value) : CUDAArray((Value) value) { }

    /// Literal (cuda.h:267-317): recorded as an immediate, never a kernel input
    CUDAArray(Value value) {
        uint64_t bits = 0;
        if constexpr (std::is_same_v<Value, bool>) bits = value ? 1 : 0;
        else memcpy(&bits, &value, sizeof(Value));
        m_index = detail::ek_append(Type, EK_OP_LITERAL, 0, 0, 0, bits);
    }

    template <typename... Args, enable_if_t<(sizeof...(Args) > 1)> = 0>
    CUDAArray(Args &&... args) {
        Value data[] = { (Value) args... };
        m_index = cuda_var_copy_to_device(Type, sizeof...(Args), data);
    }

    // ---- vertical operations (cuda.h:341-467) ----
    CUDAArray add_(const CUDAArray &v) const { return bin_(EK_OP_ADD, v); }
    CUDAArray sub_(const CUDAArray &v) const { return bin_(EK_OP_SUB, v); }
    CUDAArray mul_(const CUDAArray &v) const { return bin_(EK_OP_MUL, v); }
    CUDAArray mulhi_(const CUDAArray &v) const { return bin_(EK_OP_MULHI, v); }
    CUDAArray div_(const CUDAArray &v) const { return bin_(EK_OP_DIV, v); }
    CUDAArray mod_(const CUDAArray &v) const { return bin_(EK_OP_MOD, v); }
    CUDAArray max_(const CUDAArray &v) const { return bin_(EK_OP_MAX, v); }
    CUDAArray min_(const CUDAArray &v) const { return bin_(EK_OP_MIN, v); }
    CUDAArray xor_(const CUDAArray &v) const { return bin_(EK_OP_XOR, v); }

    CUDAArray fmadd_(const CUDAArray &a, const CUDAArray &b) const {
        return from_index_(detail::ek_append(Type, EK_OP_FMA, m_index, a.m_index, b.m_index));
    }
    CUDAArray fmsub_(const CUDAArray &a, const CUDAArray &b) const { return fmadd_(a, -b); }
    CUDAArray fnmadd_(const CUDAArray &a, const CUDAArray &b) const { return fmadd_(-a, b); }
    CUDAArray fnmsub_(const CUDAArray &a, const CUDAArray &b) const { return -fmadd_(a, b); }

    CUDAArray abs_() const { return un_(EK_OP_ABS); }
    CUDAArray neg_() const { return un_(EK_OP_NEG); }
    CUDAArray sqrt_() const { return un_(EK_OP_SQRT); }
    /// exp/log/sin/cos/rcp/rsqrt: single opcodes that evaluate the CPU path's Cephes forms
    /// (array_math.h:261-367,711-898) on the device, not the reference GPU's .approx instructions
    CUDAArray exp_() const { return un_(EK_OP_EXP); }
    CUDAArray log_() const { return un_(EK_OP_LOG); }
    CUDAArray sin_() const { return un_(EK_OP_SIN); }
    CUDAArray cos_() const { return un_(EK_OP_COS); }
    std::pair<CUDAArray, CUDAArray> sincos_() const { return { sin_(), cos_() }; }
    CUDAArray rcp_() const { return un_(EK_OP_RCP); }
    CUDAArray rsqrt_() const { return un_(EK_OP_RSQRT); }
    /// tan/cot/asin/acos/atan/atan2: single opcodes for Float32 that compute, bit for bit, what array_math.h's
    /// generic bodies (array_math.h:369-668) would record op by op.  array_math.h prefers these members when they
    /// exist; for CUDAArray<double> and integer arrays they do not, and those keep the traced bodies.
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray tan_() const { return un_(EK_OP_TAN); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray cot_() const { return un_(EK_OP_COT); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray asin_() const { return un_(EK_OP_ASIN); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray acos_() const { return un_(EK_OP_ACOS); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray atan_() const { return un_(EK_OP_ATAN); }
    /// atan2(*this, x): *this is y
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0>
    CUDAArray atan2_(const CUDAArray &x) const { return bin_(EK_OP_ATAN2, x); }
    /// sinh/cosh/tanh/asinh/acosh/atanh/cbrt: the same for the hyperbolic functions and the cube root
    /// (array_math.h:900-954,997-1348).  csch, sech and coth are rcp() of these.
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray sinh_() const { return un_(EK_OP_SINH); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray cosh_() const { return un_(EK_OP_COSH); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray tanh_() const { return un_(EK_OP_TANH); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray asinh_() const { return un_(EK_OP_ASINH); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray acosh_() const { return un_(EK_OP_ACOSH); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray atanh_() const { return un_(EK_OP_ATANH); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray cbrt_() const { return un_(EK_OP_CBRT); }
    /// sincosh (array_math.h:1067-1127) records the same operations as sinh followed by cosh, so it is the pair of them
    /// (DiffArray's sinh_ / cosh_ call it)
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0>
    std::pair<CUDAArray, CUDAArray> sincosh_() const { return { sinh_(), cosh_() }; }
    /// erf/erfc/erfinv/lgamma/tgamma: the same for the special functions (special.h:56-164,222-246,275-312).  special.h
    /// calls no members, so the free overloads of CUDAArray<float> below are the entry points that use these.
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray erf_() const { return un_(EK_OP_ERF); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray erfc_() const { return un_(EK_OP_ERFC); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray erfinv_() const { return un_(EK_OP_ERFINV); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray lgamma_() const { return un_(EK_OP_LGAMMA); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray tgamma_() const { return un_(EK_OP_TGAMMA); }
    /// pow/frexp: the same for array_math.h:682-709,956-958.  pow(x, y) with a scalar y that is an integer keeps
    /// array_math.h's repeated multiplication; any other y reaches pow_.  fmod and ldexp keep their traced bodies: on an
    /// H100 their native forms measured no faster (DESIGN.md 6).
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0>
    CUDAArray pow_(const CUDAArray &y) const { return bin_(EK_OP_POW, y); }
    /// frexp(*this): (mantissa, exponent), two nodes
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0>
    std::pair<CUDAArray, CUDAArray> frexp_() const { return { un_(EK_OP_FREXP_M), un_(EK_OP_FREXP_E) }; }
    /// hypot/dawson/erfi: called by the free overloads of CUDAArray<float> below (array_math.h:1362-1379,
    /// special.h:249-271)
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0>
    CUDAArray hypot_(const CUDAArray &b) const { return bin_(EK_OP_HYPOT, b); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray dawson_() const { return un_(EK_OP_DAWSON); }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0> CUDAArray erfi_() const { return un_(EK_OP_ERFI); }
    /// carlson_rf/carlson_rd/carlson_rc with *this as x: called by the free overloads of Array<CUDAArray<float>, N>
    /// below (special.h:325-482)
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0>
    CUDAArray carlson_rf_(const CUDAArray &y, const CUDAArray &z) const {
        return from_index_(detail::ek_append(Type, EK_OP_CARLSON_RF, m_index, y.m_index, z.m_index));
    }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0>
    CUDAArray carlson_rd_(const CUDAArray &y, const CUDAArray &z) const {
        return from_index_(detail::ek_append(Type, EK_OP_CARLSON_RD, m_index, y.m_index, z.m_index));
    }
    template <typename T = Value, enable_if_t<std::is_same_v<T, float>> = 0>
    CUDAArray carlson_rc_(const CUDAArray &y) const { return bin_(EK_OP_CARLSON_RC, y); }
    CUDAArray floor_() const { return un_(EK_OP_FLOOR); }
    CUDAArray ceil_() const { return un_(EK_OP_CEIL); }
    CUDAArray round_() const { return un_(EK_OP_ROUND); }
    CUDAArray trunc_() const { return un_(EK_OP_TRUNC); }
    template <typename T> T floor2int_() const { return T::from_index_(detail::ek_append(T::Type, EK_OP_FLOOR2INT, m_index)); }
    template <typename T> T ceil2int_() const { return T::from_index_(detail::ek_append(T::Type, EK_OP_CEIL2INT, m_index)); }

    // ---- shifts / bit operations (cuda.h:499-580); 64-bit shifts take a 32-bit count ----
    CUDAArray sl_(const CUDAArray &v) const { return bin_(EK_OP_SHL, v); }
    CUDAArray sr_(const CUDAArray &v) const { return bin_(EK_OP_SHR, v); }
    CUDAArray sl_(size_t value) const { return sl_(CUDAArray((Value) value)); }
    CUDAArray sr_(size_t value) const { return sr_(CUDAArray((Value) value)); }
    template <size_t Imm> CUDAArray sl_() const { return sl_(Imm); }
    template <size_t Imm> CUDAArray sr_() const { return sr_(Imm); }
    CUDAArray not_() const { return un_(EK_OP_NOT); }
    CUDAArray popcnt_() const { return un_(EK_OP_POPC); }
    CUDAArray lzcnt_() const { return un_(EK_OP_CLZ); }
    CUDAArray tzcnt_() const { return un_(EK_OP_CTZ); }

    /// value | mask and value & mask are select forms when the operand is a mask (cuda.h:545-572);
    /// the runtime lowers (AND|OR)(value, Bool) accordingly
    template <typename T> CUDAArray or_(const CUDAArray<T> &v) const {
        return from_index_(detail::ek_append(Type, EK_OP_OR, m_index, v.index_()));
    }
    template <typename T> CUDAArray and_(const CUDAArray<T> &v) const {
        return from_index_(detail::ek_append(Type, EK_OP_AND, m_index, v.index_()));
    }
    template <typename T> CUDAArray andnot_(const CUDAArray<T> &v) const { return and_(!v); }

    // ---- comparisons (cuda.h:582-630) ----
    MaskType gt_(const CUDAArray &v) const { return cmp_(EK_OP_GT, v); }
    MaskType ge_(const CUDAArray &v) const { return cmp_(EK_OP_GE, v); }
    MaskType lt_(const CUDAArray &v) const { return cmp_(EK_OP_LT, v); }
    MaskType le_(const CUDAArray &v) const { return cmp_(EK_OP_LE, v); }
    MaskType eq_(const CUDAArray &v) const { return cmp_(EK_OP_EQ, v); }
    MaskType neq_(const CUDAArray &v) const { return cmp_(EK_OP_NE, v); }

    static CUDAArray select_(const MaskType &m, const CUDAArray &t, const CUDAArray &f) {
        return from_index_(detail::ek_append(Type, EK_OP_SELECT, m.index_(), t.index_(), f.index_()));
    }

    // ---- initialisation (cuda.h:641-691) ----
    static CUDAArray arange_(ssize_t start, ssize_t stop, ssize_t step) {
        size_t size = size_t((stop - start + step - (step > 0 ? 1 : -1)) / step);
        using UInt32 = CUDAArray<uint32_t>;
        UInt32 index = UInt32::from_index_(detail::ek_append(EnokiType::UInt32, EK_OP_INDEX));
        index.m_index = cuda_var_set_size(index.m_index, size);
        if (start == 0 && step == 1)
            return CUDAArray(index);
        return fmadd(CUDAArray(index), CUDAArray((Value) step), CUDAArray((Value) start));
    }

    static CUDAArray linspace_(Value min, Value max, size_t size) {
        using UInt32 = CUDAArray<uint32_t>;
        UInt32 index = UInt32::from_index_(detail::ek_append(EnokiType::UInt32, EK_OP_INDEX));
        index.m_index = cuda_var_set_size(index.m_index, size);
        Value step = (max - min) / Value(size - 1);
        return fmadd(CUDAArray(index), CUDAArray(step), CUDAArray(min));
    }

    static CUDAArray empty_(size_t size) {
        return from_index_(cuda_var_register(Type, size, cuda_malloc(size * sizeof(Value)), true));
    }

    static CUDAArray zero_(size_t size) {
        if (size == 1)
            return CUDAArray(Value(0));
        void *ptr = cuda_malloc(size * sizeof(Value));
        cuda_fill((uint8_t *) ptr, 0, size * sizeof(Value));
        return from_index_(cuda_var_register(Type, size, ptr, true));
    }

    static CUDAArray full_(const Value &value, size_t size) {
        if (size == 1)
            return CUDAArray(value);
        using UInt = uint_array_t<Value>;
        void *ptr = cuda_malloc(size * sizeof(Value));
        cuda_fill((UInt *) ptr, memcpy_cast<UInt>(value), size);
        return from_index_(cuda_var_register(Type, size, ptr, true));
    }

    // ---- horizontal operations (cuda.h:693-794): lazy reductions fused into the producing sweep ----
    CUDAArray hsum_() const { return size() == 1 ? *this : un_(EK_OP_HSUM); }
    CUDAArray hprod_() const { return size() == 1 ? *this : un_(EK_OP_HPROD); }
    CUDAArray hmax_() const { return size() == 1 ? *this : un_(EK_OP_HMAX); }
    CUDAArray hmin_() const { return size() == 1 ? *this : un_(EK_OP_HMIN); }

    bool all_() const {
        if (size() == 1) return (bool) coeff(0);
        return (bool) CUDAArray<bool>::from_index_(detail::ek_append(EnokiType::Bool, EK_OP_ALL, m_index)).coeff(0);
    }
    bool any_() const {
        if (size() == 1) return (bool) coeff(0);
        return (bool) CUDAArray<bool>::from_index_(detail::ek_append(EnokiType::Bool, EK_OP_ANY, m_index)).coeff(0);
    }
    size_t count_() const {
        return (size_t) CUDAArray<uint32_t>::from_index_(detail::ek_append(EnokiType::UInt32, EK_OP_COUNT, m_index)).coeff(0);
    }

    CUDAArray reverse_() const {
        using UInt = uint_array_t<Value>;
        size_t n = size();
        if (n <= 1) return *this;
        eval();
        UInt *result = (UInt *) cuda_malloc(n * sizeof(Value));
        cuda_reverse(result, (const UInt *) cuda_var_ptr(m_index), n);
        return from_index_(cuda_var_register(Type, n, result, true));
    }

    CUDAArray psum_() const {
        size_t n = size();
        if (n <= 1) return *this;
        eval();
        Value *result = cuda_psum(n, (const Value *) cuda_var_ptr(m_index));
        return from_index_(cuda_var_register(Type, n, result, true));
    }

    template <typename Mask> CUDAArray compress_(const Mask &mask) const {
        if (mask.size() == 0)
            return CUDAArray();
        else if (size() == 1 && mask.size() != 0)
            return *this;
        else if (mask.size() != size())
            throw std::runtime_error("CUDAArray::compress_(): size mismatch!");
        eval();
        mask.eval();
        Value *ptr; size_t new_size;
        cuda_compress(size(), (const Value *) data(), (const bool *) mask.data(), &ptr, &new_size);
        return map(ptr, new_size, true);
    }

    // ---- memory (cuda.h:796-905) ----
    CUDAArray &eval() { cuda_eval_var(m_index); return *this; }
    const CUDAArray &eval() const { cuda_eval_var(m_index); return *this; }
    static CUDAArray map(void *ptr, size_t size, bool dealloc = false) { return from_index_(cuda_var_register(Type, size, ptr, dealloc)); }
    static CUDAArray copy(const void *ptr, size_t size) { return from_index_(cuda_var_copy_to_device(Type, size, ptr)); }
    CUDAArray &managed() { cuda_make_managed(m_index); return *this; }
    const CUDAArray &managed() const { cuda_make_managed(m_index); return *this; }

    // ---- DLPack (no counterpart in the reference): zero-copy exchange with libtorch (at::toDLPack / at::fromDLPack)
    //      and anything else that speaks DLPack; the rules are those of ek_dlpack_export / ek_dlpack_import
    /// A managed tensor aliasing this array (evaluated first).  `consumer_stream` is the cudaStream_t the consumer uses
    /// it on (nullptr: none); order that stream after the backend's work with ek_stream_signal_external().
    DLManagedTensor *to_dlpack(void *consumer_stream = nullptr) const {
        void *m = ek_dlpack_export(m_index, 0, consumer_stream);
        if (!m) detail::ek_throw();
        return (DLManagedTensor *) m;
    }
    DLManagedTensorVersioned *to_dlpack_versioned(void *consumer_stream = nullptr) const {
        void *m = ek_dlpack_export(m_index, 1, consumer_stream);
        if (!m) detail::ek_throw();
        return (DLManagedTensorVersioned *) m;
    }
    /// An array aliasing `t`, which it owns from here on: the deleter runs once the backend's last use of the buffer
    /// has completed.  A refused tensor (device, dtype other than this array's, layout, size) stays the caller's.
    static CUDAArray from_dlpack(DLManagedTensor *t) { return from_dlpack_(t, t ? &t->dl_tensor : nullptr, 0); }
    static CUDAArray from_dlpack(DLManagedTensorVersioned *t) { return from_dlpack_(t, t ? &t->dl_tensor : nullptr, 1); }

    template <size_t Stride, typename Index, typename Mask>
    static CUDAArray gather_(const void *ptr_, const Index &index, const Mask &mask) {
        uint32_t ptr = cuda_var_register_ptr(ptr_);
        uint32_t r;
        try { r = detail::ek_append(Type, EK_OP_GATHER, ptr, index.index_(), mask.index_(), (uint64_t) Stride); }
        catch (...) { ek_dec_ref_ext(ptr); throw; }
        ek_dec_ref_ext(ptr);
        return from_index_(r);
    }

    template <size_t Stride, typename Index, typename Mask>
    ENOKI_INLINE void scatter_(void *ptr_, const Index &index, const Mask &mask) const {
        scatter_impl_<Stride>(EK_OP_SCATTER, ptr_, index, mask);
    }

    template <size_t Stride, typename Index, typename Mask>
    void scatter_add_(void *ptr_, const Index &index, const Mask &mask) const {
        scatter_impl_<Stride>(EK_OP_SCATTER_ADD, ptr_, index, mask);
    }

    auto operator->() const {
        using BaseType = std::decay_t<std::remove_pointer_t<Value>>;
        return call_support<BaseType, CUDAArray>(*this);
    }

    /// Virtual-call dispatch support (cuda.h:814-843): (instance pointer, indices that refer to it), pointers ascending,
    /// indices ascending; cached per array like the reference's.
    /// (ek_partition: hash + radix grouping on the device up to 65 536 distinct pointers, host-side stable sort above,
    /// see ek_partition.cu.)
    template <typename T = Value, enable_if_t<std::is_pointer_v<T> || std::is_same_v<T, uintptr_t>> = 0>
    std::vector<std::pair<Value, CUDAArray<uint32_t>>> partition_() const {
        using Groups = std::vector<std::pair<Value, CUDAArray<uint32_t>>>;
        if (m_cached_partition)
            return *m_cached_partition;
        eval();
        /* ek_partition hands back: pinned-host instance pointers and counts (counts[0] = number of groups), and a
           malloc'd array of device index lists, one per group (ownership as horiz.cu:83-121) */
        void **instances = nullptr; uint32_t *sizes = nullptr; uint32_t **lists = nullptr;
        cuda_partition(size(), (const void **) data(), &instances, &sizes, &lists);
        Groups *groups = new Groups();
        const uint32_t n_groups = sizes[0];
        groups->reserve(n_groups);
        for (uint32_t g = 0; g < n_groups; ++g) {
            uint32_t handle = cuda_var_register(EnokiType::UInt32, sizes[g + 1], lists[g], /* dealloc = */ true);
            groups->emplace_back((Value) instances[g], CUDAArray<uint32_t>::from_index_(handle));
        }
        cuda_host_free(instances); cuda_host_free(sizes); free(lists);
        m_cached_partition = groups;
        return *groups;
    }

    static CUDAArray from_dlpack_(void *managed, const DLTensor *t, int versioned) {
        const int k = (int) Type;          /* EnokiType: Int8 = 1, UInt8, Int16, ..., UInt64 = 8, Float16 .. Float64, Bool */
        const uint8_t code = k <= 8 ? (k % 2 ? kDLInt : kDLUInt) : Type == EnokiType::Bool ? kDLBool : kDLFloat;
        if (t && (t->dtype.code != code || t->dtype.bits != 8 * sizeof(Value)))
            throw std::runtime_error("CUDAArray::from_dlpack(): the tensor's dtype (code " + std::to_string(t->dtype.code) +
                                     ", " + std::to_string(t->dtype.bits) + " bits) is not this array's");
        return from_index_(detail::ek_chk(ek_dlpack_import(managed, versioned)));
    }

    Index index_() const { return m_index; }
    /* the name the reference's cuda_printf template reads the handle by (array_router.h:973) */
    Index index() const { return m_index; }
    size_t size() const { return m_index ? cuda_var_size(m_index) : 0; }
    bool empty() const { return size() == 0; }
    const Value *data() const { return (const Value *) cuda_var_ptr(m_index); }
    Value *data() { return (Value *) cuda_var_ptr(m_index); }
    void resize(size_t size) { m_index = cuda_var_set_size(m_index, size, true); }

    Value coeff(size_t i) const {
        Value result = (Value) 0;
        cuda_fetch_element(&result, m_index, i, sizeof(Value));
        return result;
    }

    static CUDAArray from_index_(Index index) {
        CUDAArray a;
        a.m_index = index;
        return a;
    }

protected:
    CUDAArray un_(ek_op op) const { return from_index_(detail::ek_append(Type, op, m_index)); }
    CUDAArray bin_(ek_op op, const CUDAArray &v) const { return from_index_(detail::ek_append(Type, op, m_index, v.m_index)); }
    MaskType cmp_(ek_op op, const CUDAArray &v) const {
        return MaskType::from_index_(detail::ek_append(EnokiType::Bool, op, m_index, v.m_index));
    }
    template <size_t Stride, typename Index, typename Mask>
    void scatter_impl_(ek_op op, void *ptr_, const Index &index, const Mask &mask) const {
        uint32_t ptr = cuda_var_register_ptr(ptr_);
        uint32_t var = ek_trace_append(op == EK_OP_SCATTER ? EK_UINT64 : (ek_type) Type, op, ptr, index.index_(), mask.index_(),
                                       ((uint64_t) Stride << 32) | m_index);
        ek_dec_ref_ext(ptr);
        cuda_var_mark_side_effect(detail::ek_chk(var));
    }

    /* Same object layout as the reference (cuda.h:951-953): the handle plus the cached partition of pointer arrays.
       The size is part of the contract -- header templates size their recursion by sizeof(Value), e.g. morton.h:56,
       77 (`Level = clog2i(sizeof(Value) * 8)`): with a 4-byte object the 64-bit Morton decode loses its last step. */
    Index m_index = 0;
    mutable std::vector<std::pair<Value, CUDAArray<uint32_t>>> *m_cached_partition = nullptr;
};
static_assert(sizeof(CUDAArray<float>) == 16, "CUDAArray<T> must keep the reference's 16-byte layout");

/// special.h's erf, erfc, erfinv, lgamma and tgamma are free templates.  These non-template overloads are exact matches
/// for a CUDAArray<float>, so they win over the templates, and argument-dependent lookup finds them whichever of the two
/// headers comes first.  erf<FloatC>(x) with explicit template arguments still records special.h's body op by op, and
/// DiffArray, nested arrays and CUDAArray<double> keep the templates.
inline CUDAArray<float> erf(const CUDAArray<float> &x) { return x.erf_(); }
inline CUDAArray<float> erfc(const CUDAArray<float> &x) { return x.erfc_(); }
inline CUDAArray<float> erfinv(const CUDAArray<float> &x) { return x.erfinv_(); }
inline CUDAArray<float> lgamma(const CUDAArray<float> &x) { return x.lgamma_(); }
inline CUDAArray<float> tgamma(const CUDAArray<float> &x) { return x.tgamma_(); }
/// The same for array_math.h's free template hypot and special.h's dawson and erfi.  Only a call whose operands are all
/// CUDAArray<float> matches: a mixed call such as hypot(x, 1.f) still takes array_math.h's template and records its body
/// op by op.  erfi<FloatC>(x) calls dawson unqualified, so its traced body uses the native dawson.
inline CUDAArray<float> hypot(const CUDAArray<float> &a, const CUDAArray<float> &b) { return a.hypot_(b); }
inline CUDAArray<float> dawson(const CUDAArray<float> &x) { return x.dawson_(); }
inline CUDAArray<float> erfi(const CUDAArray<float> &x) { return x.erfi_(); }
/// special.h's Carlson integrals take one vector: these overloads match exactly Array<CUDAArray<float>, 3> (carlson_rf,
/// carlson_rd) and Array<CUDAArray<float>, 2> (carlson_rc), which is what comp_ellint_1/2 and ellint_1/2 build and what
/// carlson_rj passes to carlson_rc, so those pick them up.  Each is one node: the duplication loop runs per element on
/// the device instead of on the host with one synchronisation per pass (DESIGN.md 4).  The templates' assert on the
/// argument domain is not evaluated here (it would cost an evaluation and a synchronisation of its own); arguments
/// outside it give what the traced body gives.  DiffArray, CUDAArray<double>, types derived from Array and calls with
/// explicit template arguments keep the templates.
inline CUDAArray<float> carlson_rf(const Array<CUDAArray<float>, 3> &xyz) { return xyz.x().carlson_rf_(xyz.y(), xyz.z()); }
inline CUDAArray<float> carlson_rd(const Array<CUDAArray<float>, 3> &xyz) { return xyz.x().carlson_rd_(xyz.y(), xyz.z()); }
inline CUDAArray<float> carlson_rc(const Array<CUDAArray<float>, 2> &xy) { return xy.x().carlson_rc_(xy.y()); }

template <typename T, enable_if_t<!is_diff_array_v<T> && is_cuda_array_v<T>> = 0>
ENOKI_INLINE void set_label(const T &a, const char *label) {
    if constexpr (array_depth_v<T> >= 2) {
        for (size_t i = 0; i < T::Size; ++i)
            set_label(a.coeff(i), (std::string(label) + "." + std::to_string(i)).c_str());
    } else {
        cuda_var_set_label(a.index_(), label);
    }
}

/// STL allocators over unified / pinned memory (cuda.h:966-1010)
template <typename T> class cuda_managed_allocator {
public:
    using value_type = T;
    cuda_managed_allocator() = default;
    template <typename T2> cuda_managed_allocator(const cuda_managed_allocator<T2> &) { }
    value_type *allocate(size_t n) { return (value_type *) cuda_managed_malloc(n * sizeof(T)); }
    void deallocate(value_type *ptr, size_t) { cuda_free(ptr); }
    bool operator==(const cuda_managed_allocator &) { return true; }
    bool operator!=(const cuda_managed_allocator &) { return false; }
};

template <typename T> class cuda_host_allocator {
public:
    using value_type = T;
    cuda_host_allocator() = default;
    template <typename T2> cuda_host_allocator(const cuda_host_allocator<T2> &) { }
    value_type *allocate(size_t n) { return (value_type *) cuda_host_malloc(n * sizeof(T)); }
    void deallocate(value_type *ptr, size_t) { cuda_host_free(ptr); }
    bool operator==(const cuda_host_allocator &) { return true; }
    bool operator!=(const cuda_host_allocator &) { return false; }
};

NAMESPACE_END(enoki)

#if defined(ENOKI_AUTODIFF_H)
#  include <enoki/autodiff_b200.h>
#endif
