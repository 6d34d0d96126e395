/*
 * ek_internal.h -- host-side data structures of the runtime (not part of the ABI).
 *
 * Mirrors the roles of the reference's `Variable` / `Context`
 * (src/cuda/jit.cu:61-111,149-262) with dense storage (vector + free list instead
 * of unordered_map<uint32_t, Variable>) and opcodes instead of PTX strings.
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include <set>
#include <map>
#include <unordered_map>
#include <memory>
#include <atomic>
#include "../../include/enoki_b200.h"
#include "ek_isa.h"

#define EK_REG_RESERVED 10u     /* jit.cu:43 ENOKI_CUDA_REG_RESERVED: handles 1..9 are reserved */

struct EkVariable {
    ek_type  type = EK_INVALID;
    ek_op    op = EK_OP_INVALID;
    uint32_t dep[4] = { 0, 0, 0, 0 };   /* dep[3]: value operand of scatter/scatter_add      */
    uint32_t extra_dep = 0;             /* scatter/gather operand kept alive (jit.cu:88-89) */
    uint64_t imm = 0;
    size_t   size = 0;
    void    *data = nullptr;
    uint32_t ref_ext = 0, ref_int = 0;
    uint32_t subtree_size = 0;
    uint64_t seq = 0;                   /* creation order (handles are recycled, so a handle says nothing about age) */
    bool side_effect = false;
    bool dirty = false;
    bool free_data = true;
    bool direct_pointer = false;
    bool used = false;                  /* slot in use */
    std::string *label = nullptr;
    std::string *fmt = nullptr;         /* format of a print node (EK_OP_PRINTF), owned with it */
    void *dlpack = nullptr;             /* imported DLPack tensor that owns `data` (ek_dlpack.cpp); free_data is false */
    bool dlpack_versioned = false;
};

struct EkProgramCacheEntry {
    std::vector<uint8_t> key;
    EkInstr  *d_prog = nullptr;
    uint32_t *d_lit = nullptr;
};

struct EkContext {
    bool initialized = false;
    int device = 0;
    int num_sms = 132;
    size_t smem_optin = 227 * 1024;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev_start = nullptr, ev_stop = nullptr;     /* per-launch timing */
    cudaEvent_t tm_start = nullptr, tm_stop = nullptr;     /* user timer        */
    bool timing = false;
    uint32_t log_level = 0;

    std::vector<EkVariable> vars;       /* index = handle */
    std::vector<uint32_t> free_handles;
    std::set<uint32_t> live;            /* jit.cu:166-167 */
    uint64_t next_seq = 1;              /* EkVariable::seq counter */
    int fast_mode = 1;                  /* 32-bit fast sweep kernel: 1 = use it, 0 = general kernels only (ek_set_fast_mode;
                                           ek_init() leaves it as it is) */
    std::vector<uint32_t> dirty;        /* jit.cu:169-170 */
    std::unordered_map<const void *, uint32_t> ptr_map;    /* jit.cu:178-179 */
    uint32_t scatter_gather_operand = 0;
    std::vector<std::pair<void (*)(void *), void *>> callbacks;
    /* work that was recorded but not launched yet (batched adjoint levels): must reach the stream before the
       allocator synchronises and trims, because that work may still read blocks on the free list */
    cudaStream_t d2h_stream = nullptr;          /* read-back stream of ek_memcpy_from_device_overlapped() */
    cudaEvent_t d2h_event = nullptr;
    cudaEvent_t handoff_event = nullptr;        /* ek_stream_wait_external / ek_stream_signal_external */
    void (*pre_trim_hook)(void *) = nullptr;
    void *pre_trim_arg = nullptr;

    /* allocator (jit.cu:1636-1896): exact-size free lists, stream ordered */
    std::unordered_map<void *, size_t> alloc_size;          /* device + managed */
    std::unordered_map<void *, int> alloc_kind;             /* 0 device, 1 managed, 2 host */
    std::map<std::pair<int, size_t>, std::vector<void *>> free_lists;
    size_t used = 0, watermark = 0, cached = 0;

    /* program cache */
    std::unordered_map<uint64_t, std::vector<EkProgramCacheEntry>> programs;

    /* reduction scratch */
    uint64_t *red_partials = nullptr;   /* [EK_MAX_RED][max_grid] */
    uint32_t *red_counters = nullptr;
    uint32_t max_grid = 0;

    /* L2 flush scratch */
    void *flush_buf = nullptr;
    size_t flush_bytes = 0;

    ek_stats stats = {};
};

#define EK_MAX_RED 32

EkContext &ek_ctx();
void ek_set_error(const std::string &msg);
void ek_cuda_check_impl(cudaError_t err, const char *file, int line);
#define ek_cuda_check(x) ek_cuda_check_impl((x), __FILE__, __LINE__)

/* DLPack releases (ek_dlpack.cpp).  ek_dlpack_pending counts queued releases: exported tensors dropped on any thread
   and freed imports whose producer has not been told yet.  Entry points call ek_dlpack_drain(), one atomic load when
   nothing is queued; `wait` (ek_sync, ek_shutdown) waits for every freed import's last use and releases it. */
extern std::atomic<uint32_t> ek_dlpack_pending;
void ek_dlpack_drain_slow(bool wait);
static inline void ek_dlpack_drain(bool wait = false) {
    if (ek_dlpack_pending.load(std::memory_order_acquire)) ek_dlpack_drain_slow(wait);
}
/* queue the release of a freed variable's imported tensor (called by var_free on the owning thread) */
void ek_dlpack_release_import(EkVariable &v);
/* ek_shutdown: wait for and release every queued tensor; exports still held by consumers are forgotten */
void ek_dlpack_shutdown();
/* the device ek_init() runs on, or will pick */
int ek_planned_device();

/* kernels (defined in .cu files) */
/* trig: the body contains an operation of the extension instantiations (ek_isa.h ek_dop_ext: tan ... carlson_rc) */
cudaError_t ek_launch_sweep(int V, bool inline_prog, bool trig, const EkSweepArgs &args, unsigned grid, unsigned block,
                            size_t smem_bytes, cudaStream_t stream);
/* 32-bit fast kernel (ek_sweep_fast.cu): args.prog_inline holds the lowered program; block = 128 or 256 */
cudaError_t ek_launch_sweep_fast(const EkSweepArgs &args, unsigned grid, unsigned block, size_t smem_bytes, cudaStream_t stream);
void ek_launch_fill(void *ptr, size_t elem_size, uint64_t value, size_t n, cudaStream_t stream);
void ek_launch_reverse(void *out, const void *in, size_t elem_size, size_t n, cudaStream_t stream);
void ek_launch_flush(void *buf, size_t bytes, cudaStream_t stream);
/* inclusive prefix sum of n uint32 values on the runtime's stream (ek_scan.cu: the three-phase scan of ek_psum) */
void ek_scan_incl_u32(const uint32_t *in, uint32_t *out, size_t n);

/* type helpers */
static inline size_t ek_type_size(ek_type t) {
    switch (t) {
        case EK_INT8: case EK_UINT8: case EK_BOOL: return 1;
        case EK_INT16: case EK_UINT16: case EK_FLOAT16: return 2;
        case EK_INT32: case EK_UINT32: case EK_FLOAT32: return 4;
        case EK_INT64: case EK_UINT64: case EK_FLOAT64: case EK_POINTER: return 8;
        default: return 0;
    }
}
static inline bool ek_is_float(ek_type t) { return t == EK_FLOAT16 || t == EK_FLOAT32 || t == EK_FLOAT64; }
static inline bool ek_is_signed(ek_type t) {
    return t == EK_INT8 || t == EK_INT16 || t == EK_INT32 || t == EK_INT64 || ek_is_float(t);
}
static inline bool ek_is_64(ek_type t) { return ek_type_size(t) == 8; }
const char *ek_type_name(ek_type t);
const char *ek_op_name(ek_op op);
/* element-wise operations of one and of two operands (the trigonometric, hyperbolic, special and remaining Float32
   math ones come after EK_OP_PRINTF) */
static inline bool ek_op_unary(ek_op op) {
    return (op >= EK_OP_MOV && op <= EK_OP_CTZ) || (op >= EK_OP_TAN && op <= EK_OP_ATAN) || (op >= EK_OP_SINH && op <= EK_OP_TGAMMA) ||
           op == EK_OP_FREXP_M || op == EK_OP_FREXP_E || op == EK_OP_DAWSON || op == EK_OP_ERFI;
}
static inline bool ek_op_binary(ek_op op) {
    return (op >= EK_OP_ADD && op <= EK_OP_MUL_NZ) || op == EK_OP_ATAN2 || op == EK_OP_POW || op == EK_OP_HYPOT ||
           op == EK_OP_CARLSON_RC;
}
/* the ternary Carlson integrals (x, y, z): only x is read from the accumulator */
static inline bool ek_op_carlson3(ek_op op) { return op == EK_OP_CARLSON_RF || op == EK_OP_CARLSON_RD; }

/* cuda_printf formats (ek_printf.cpp).  A parsed format is a list of segments: literal text (conv == 0, "%%" already
   reduced to "%") or one conversion, `text` being its spec as written ("%-08.3lx") and `arg` the argument it takes. */
struct EkPrintSeg { std::string text; char conv; uint8_t len; /* 0 none, 1 hh, 2 h, 3 l, 4 ll */ uint8_t arg; };
/* check `fmt` against the argument types; false (and `err`) when it is rejected */
bool ek_printf_parse(const char *fmt, uint32_t narg, const ek_type *types, std::vector<EkPrintSeg> &segs, std::string &err);
/* append one element's line: bits[k] = raw bits of argument k for that element (zero-extended) */
void ek_printf_append(std::string &out, const std::vector<EkPrintSeg> &segs, const ek_type *types, const uint64_t *bits);
