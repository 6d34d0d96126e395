/*
 * ek_eval.cpp -- scheduler + sweep-program assembler + launcher (cuda_eval).
 *
 * Behavioural spec: src/cuda/jit.cu:1385-1508 (sweep_recursive / cuda_eval) and
 * :983-1227 (cuda_jit_assemble) of the reference:
 *   - live roots are grouped by array size, scheduled DFS post-order with the
 *     heavier subtree first, one kernel per group;
 *   - a variable is STORED by a kernel iff it is externally referenced, has no
 *     side effect and has the sweep's size (jit.cu:1027-1030,1165-1169);
 *   - after evaluation the dependencies of stored variables are dropped
 *     (jit.cu:1484-1507).
 * New here:
 *   - the group program is a list of EkInstr (ek_isa.h) for ek_sweep_kernel
 *     instead of PTX text; a linear-scan allocator maps values to shared-memory
 *     slots, forwarding single-use values through registers;
 *   - "phases": horizontal reductions are lazy size-1 variables computed as an
 *     epilogue of the sweep that produces their operand; consumers of a reduction
 *     (and wide consumers of a computed size-1 value) are scheduled in a later
 *     phase, so `x / hsum(x)` needs no host round trip.
 */
#include "ek_internal.h"
static_assert(sizeof(EkSweepArgs) <= 32000, "EkSweepArgs must fit the 32 KB kernel parameter space (CUDA >= 12.1, sm_70+)");
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <sstream>
#include <unordered_set>
#include <memory>

namespace {

inline bool is_reduce(ek_op op) { return op >= EK_OP_HSUM && op <= EK_OP_COUNT; }

struct Loc {
    enum Kind : uint8_t { NONE, UNI, STAGED, SLOT, PENDING } kind = NONE;
    uint16_t idx = 0;       /* uniform word / staged unit / slot */
};

struct Group {
    uint32_t phase = 0;
    size_t size = 0;
    std::vector<uint32_t> roots;
    std::vector<uint32_t> sched;
    std::unordered_set<uint32_t> visited;
    std::unordered_set<uint32_t> boundary;    /* inputs produced by an earlier launch of the same eval */
};

struct Output { uint32_t var; uint32_t argw; size_t bytes; };

struct Assembled {
    std::vector<EkInstr> init, body, fini;
    std::vector<uint32_t> lits;
    std::vector<uint32_t> argw;                 /* pointer words are patched at launch */
    struct PtrFix { uint32_t argw; uint32_t var; bool output; };
    std::vector<PtrFix> ptr_fix;                /* argw index <- data pointer of var */
    std::vector<Output> outputs;                /* variables that receive storage    */
    struct Staged { uint32_t var; uint16_t unit; uint8_t esize; };
    std::vector<Staged> staged;
    struct Scalar { uint32_t var; };
    std::vector<Scalar> scalars;
    uint32_t n_tmp = 0, n_in_units = 0, n_red = 0;
    uint32_t extra_bytes = 0;
    uint32_t n_arith = 0;
    bool has64 = false;                         /* any 64-bit value: needs the general (high-plane) kernel */
    uint32_t release_mask = 0;                  /* staged inputs (bit k: staged[k]) dead after body[release_at] ... */
    int release_at = -1;                        /* ... where the fast kernel's lowering inserts its FF_REL instruction (early release) */
    uint64_t bytes_in = 0, bytes_out = 0;
    struct DescFix { uint32_t argw; uint32_t count_limit; };
    /* shared-memory 'extra' region: staged gather tables and privatised scatter_add bins; the offsets / copy counts
       written into the descriptors at assembly time are the general kernels' layout -- the fast kernel re-lays the
       region out for its block size (layout_extra) */
    struct ExtraItem { uint32_t di; uint32_t count; uint8_t kind; };   /* kind 0 table, 1 float bins, 2 integer bins */
    std::vector<ExtraItem> extra_items;
    bool fast_ok = false;                       /* (programs without 64-bit values) every instruction has a fast-kernel form:
                                                   lower_fast, which takes the fast kernel's operation set from fop_of */
    uint32_t fast_len = 0;                      /* number of lowered instructions */
    std::string error;
    bool resource_error = false;     /* a limit was hit: the caller may split the group and retry */
};

#define EK_STAGE_UNIT_BUDGET 8u     /* slot units of TMA-staged inputs per pipeline stage */

/* V = elements per thread: 16 on the fast kernel, 8 or 4 on the general kernel (ek_sweep.cu) */
struct Config { int V; uint32_t T; uint32_t stages; uint32_t ctas_per_sm; size_t smem; uint32_t off_bar, off_prog, off_extra, off_slots; bool prog_in_smem;
                bool fast = false;   /* the 32-bit fast kernel (ek_sweep_fast.cu) with its own program form and extra-region layout */ };

/* ------------------------------------------------------------------ device opcode selection */
enum Cls { C_F32, C_F64, C_I32, C_U32, C_I64, C_U64, C_BAD };

Cls cls_of(ek_type t) {
    switch (t) {
        case EK_FLOAT32: return C_F32;
        case EK_FLOAT64: return C_F64;
        case EK_INT8: case EK_INT16: case EK_INT32: return C_I32;
        case EK_UINT8: case EK_UINT16: case EK_UINT32: case EK_BOOL: return C_U32;
        case EK_FLOAT16: return C_U32;     /* its binary16 bits, moved like UInt16 (emit_var refuses arithmetic on them) */
        case EK_INT64: return C_I64;
        case EK_UINT64: case EK_POINTER: return C_U64;
        default: return C_BAD;
    }
}

/* normalisation op that brings a 32-bit register back into the value range of a narrow type */
int norm_op(ek_type t) {
    switch (t) {
        case EK_INT8: return DOP_SEXT8;
        case EK_UINT8: return DOP_ZEXT8;
        case EK_INT16: return DOP_SEXT16;
        case EK_UINT16: return DOP_ZEXT16;
        default: return -1;
    }
}

/* the 32-bit register word of a value of type t with the given bits: a narrow value sign- or zero-extended from the
   type's width (as the sweep kernels hold it and load scalars), whatever lies above those bits */
uint32_t register_word(ek_type t, uint64_t bits) {
    switch (t) {
        case EK_INT8: return (uint32_t) (int32_t) (int8_t) bits;
        case EK_UINT8: return (uint32_t) (uint8_t) bits;
        case EK_INT16: return (uint32_t) (int32_t) (int16_t) bits;
        case EK_UINT16: case EK_FLOAT16: return (uint32_t) (uint16_t) bits;
        default: return (uint32_t) bits;
    }
}

#define SEL(f32, f64, i32, u32, i64, u64) \
    (c == C_F32 ? (f32) : c == C_F64 ? (f64) : c == C_I32 ? (i32) : c == C_U32 ? (u32) : c == C_I64 ? (i64) : (u64))

/* returns device opcode or -1 */
int pick_op(ek_op op, ek_type vt, ek_type at /* operand type */) {
    Cls c = cls_of(op >= EK_OP_GT && op <= EK_OP_NE ? at : vt);
    if (c == C_BAD) return -1;
    switch (op) {
        case EK_OP_MOV:   return SEL(DOP_LOAD_32, DOP_LOAD_64, DOP_LOAD_32, DOP_LOAD_32, DOP_LOAD_64, DOP_LOAD_64);
        case EK_OP_NEG:   return SEL(DOP_NEG_F32, DOP_NEG_F64, DOP_NEG_I32, DOP_NEG_I32, DOP_NEG_I64, DOP_NEG_I64);
        case EK_OP_ABS:   return SEL(DOP_ABS_F32, DOP_ABS_F64, DOP_ABS_I32, DOP_LOAD_32, DOP_ABS_I64, DOP_LOAD_64);
        case EK_OP_SQRT:  return SEL(DOP_SQRT_F32, DOP_SQRT_F64, -1, -1, -1, -1);
        case EK_OP_RCP:   return SEL(DOP_RCP_F32, DOP_RCP_F64, -1, -1, -1, -1);
        case EK_OP_RSQRT: return SEL(DOP_RSQRT_F32, DOP_RSQRT_F64, -1, -1, -1, -1);
        case EK_OP_EXP:   return SEL(DOP_EXP_F32, DOP_EXP_F64, -1, -1, -1, -1);
        case EK_OP_LOG:   return SEL(DOP_LOG_F32, DOP_LOG_F64, -1, -1, -1, -1);
        case EK_OP_SIN:   return SEL(DOP_SIN_F32, DOP_SIN_F64, -1, -1, -1, -1);
        case EK_OP_COS:   return SEL(DOP_COS_F32, DOP_COS_F64, -1, -1, -1, -1);
        case EK_OP_TAN:   return SEL(DOP_TAN_F32, -1, -1, -1, -1, -1);
        case EK_OP_COT:   return SEL(DOP_COT_F32, -1, -1, -1, -1, -1);
        case EK_OP_ASIN:  return SEL(DOP_ASIN_F32, -1, -1, -1, -1, -1);
        case EK_OP_ACOS:  return SEL(DOP_ACOS_F32, -1, -1, -1, -1, -1);
        case EK_OP_ATAN:  return SEL(DOP_ATAN_F32, -1, -1, -1, -1, -1);
        case EK_OP_ATAN2: return SEL(DOP_ATAN2_F32, -1, -1, -1, -1, -1);
        case EK_OP_SINH:  return SEL(DOP_SINH_F32, -1, -1, -1, -1, -1);
        case EK_OP_COSH:  return SEL(DOP_COSH_F32, -1, -1, -1, -1, -1);
        case EK_OP_TANH:  return SEL(DOP_TANH_F32, -1, -1, -1, -1, -1);
        case EK_OP_ASINH: return SEL(DOP_ASINH_F32, -1, -1, -1, -1, -1);
        case EK_OP_ACOSH: return SEL(DOP_ACOSH_F32, -1, -1, -1, -1, -1);
        case EK_OP_ATANH: return SEL(DOP_ATANH_F32, -1, -1, -1, -1, -1);
        case EK_OP_CBRT:  return SEL(DOP_CBRT_F32, -1, -1, -1, -1, -1);
        case EK_OP_ERF:    return SEL(DOP_ERF_F32, -1, -1, -1, -1, -1);
        case EK_OP_ERFC:   return SEL(DOP_ERFC_F32, -1, -1, -1, -1, -1);
        case EK_OP_ERFINV: return SEL(DOP_ERFINV_F32, -1, -1, -1, -1, -1);
        case EK_OP_LGAMMA: return SEL(DOP_LGAMMA_F32, -1, -1, -1, -1, -1);
        case EK_OP_TGAMMA: return SEL(DOP_TGAMMA_F32, -1, -1, -1, -1, -1);
        case EK_OP_POW:     return SEL(DOP_POW_F32, -1, -1, -1, -1, -1);
        case EK_OP_FREXP_M: return SEL(DOP_FREXP_M_F32, -1, -1, -1, -1, -1);
        case EK_OP_FREXP_E: return SEL(DOP_FREXP_E_F32, -1, -1, -1, -1, -1);
        case EK_OP_HYPOT:   return SEL(DOP_HYPOT_F32, -1, -1, -1, -1, -1);
        case EK_OP_DAWSON:  return SEL(DOP_DAWSON_F32, -1, -1, -1, -1, -1);
        case EK_OP_ERFI:    return SEL(DOP_ERFI_F32, -1, -1, -1, -1, -1);
        case EK_OP_CARLSON_RF: return SEL(DOP_CARLSON_RF_F32, -1, -1, -1, -1, -1);
        case EK_OP_CARLSON_RD: return SEL(DOP_CARLSON_RD_F32, -1, -1, -1, -1, -1);
        case EK_OP_CARLSON_RC: return SEL(DOP_CARLSON_RC_F32, -1, -1, -1, -1, -1);
        case EK_OP_FLOOR: return SEL(DOP_FLOOR_F32, DOP_FLOOR_F64, DOP_LOAD_32, DOP_LOAD_32, DOP_LOAD_64, DOP_LOAD_64);
        case EK_OP_CEIL:  return SEL(DOP_CEIL_F32, DOP_CEIL_F64, DOP_LOAD_32, DOP_LOAD_32, DOP_LOAD_64, DOP_LOAD_64);
        case EK_OP_ROUND: return SEL(DOP_ROUND_F32, DOP_ROUND_F64, DOP_LOAD_32, DOP_LOAD_32, DOP_LOAD_64, DOP_LOAD_64);
        case EK_OP_TRUNC: return SEL(DOP_TRUNC_F32, DOP_TRUNC_F64, DOP_LOAD_32, DOP_LOAD_32, DOP_LOAD_64, DOP_LOAD_64);
        case EK_OP_NOT:   return vt == EK_BOOL ? DOP_NOT_B : SEL(DOP_NOT_32, DOP_NOT_64, DOP_NOT_32, DOP_NOT_32, DOP_NOT_64, DOP_NOT_64);
        case EK_OP_POPC:  return SEL(-1, -1, DOP_POPC_32, DOP_POPC_32, DOP_POPC_64, DOP_POPC_64);
        case EK_OP_CLZ:   return SEL(-1, -1, DOP_CLZ_32, DOP_CLZ_32, DOP_CLZ_64, DOP_CLZ_64);
        case EK_OP_CTZ:   return SEL(-1, -1, DOP_CTZ_32, DOP_CTZ_32, DOP_CTZ_64, DOP_CTZ_64);
        case EK_OP_ADD:   return SEL(DOP_ADD_F32, DOP_ADD_F64, DOP_ADD_I32, DOP_ADD_I32, DOP_ADD_I64, DOP_ADD_I64);
        case EK_OP_SUB:   return SEL(DOP_SUB_F32, DOP_SUB_F64, DOP_SUB_I32, DOP_SUB_I32, DOP_SUB_I64, DOP_SUB_I64);
        case EK_OP_MUL:   return SEL(DOP_MUL_F32, DOP_MUL_F64, DOP_MUL_I32, DOP_MUL_I32, DOP_MUL_I64, DOP_MUL_I64);
        case EK_OP_MULHI: return SEL(-1, -1, DOP_MULHI_I32, DOP_MULHI_U32, DOP_MULHI_I64, DOP_MULHI_U64);
        case EK_OP_DIV:   return SEL(DOP_DIV_F32, DOP_DIV_F64, DOP_DIV_I32, DOP_DIV_U32, DOP_DIV_I64, DOP_DIV_U64);
        case EK_OP_MOD:   return SEL(-1, -1, DOP_MOD_I32, DOP_MOD_U32, DOP_MOD_I64, DOP_MOD_U64);
        case EK_OP_MIN:   return SEL(DOP_MIN_F32, DOP_MIN_F64, DOP_MIN_I32, DOP_MIN_U32, DOP_MIN_I64, DOP_MIN_U64);
        case EK_OP_MAX:   return SEL(DOP_MAX_F32, DOP_MAX_F64, DOP_MAX_I32, DOP_MAX_U32, DOP_MAX_I64, DOP_MAX_U64);
        case EK_OP_SHL:   return SEL(-1, -1, DOP_SHL_32, DOP_SHL_32, DOP_SHL_64, DOP_SHL_64);
        case EK_OP_SHR:   return SEL(-1, -1, DOP_SHR_I32, DOP_SHR_U32, DOP_SHR_I64, DOP_SHR_U64);
        case EK_OP_AND:   return SEL(DOP_AND_32, DOP_AND_64, DOP_AND_32, DOP_AND_32, DOP_AND_64, DOP_AND_64);
        case EK_OP_OR:    return SEL(DOP_OR_32, DOP_OR_64, DOP_OR_32, DOP_OR_32, DOP_OR_64, DOP_OR_64);
        case EK_OP_XOR:   return SEL(DOP_XOR_32, DOP_XOR_64, DOP_XOR_32, DOP_XOR_32, DOP_XOR_64, DOP_XOR_64);
        case EK_OP_GT:    return SEL(DOP_GT_F32, DOP_GT_F64, DOP_GT_I32, DOP_GT_U32, DOP_GT_I64, DOP_GT_U64);
        case EK_OP_GE:    return SEL(DOP_GE_F32, DOP_GE_F64, DOP_GE_I32, DOP_GE_U32, DOP_GE_I64, DOP_GE_U64);
        case EK_OP_LT:    return SEL(DOP_LT_F32, DOP_LT_F64, DOP_LT_I32, DOP_LT_U32, DOP_LT_I64, DOP_LT_U64);
        case EK_OP_LE:    return SEL(DOP_LE_F32, DOP_LE_F64, DOP_LE_I32, DOP_LE_U32, DOP_LE_I64, DOP_LE_U64);
        case EK_OP_EQ:    return SEL(DOP_EQ_F32, DOP_EQ_F64, DOP_EQ_32, DOP_EQ_32, DOP_EQ_64, DOP_EQ_64);
        case EK_OP_NE:    return SEL(DOP_NE_F32, DOP_NE_F64, DOP_NE_32, DOP_NE_32, DOP_NE_64, DOP_NE_64);
        case EK_OP_MUL_NZ: return SEL(DOP_MULNZ_F32, DOP_MULNZ_F64, -1, -1, -1, -1);
        case EK_OP_FMA:   return SEL(DOP_FMA_F32, DOP_FMA_F64, DOP_MAD_I32, DOP_MAD_I32, DOP_MAD_I64, DOP_MAD_I64);
        case EK_OP_FMA_NZ: return SEL(DOP_FMANZ_F32, DOP_FMANZ_F64, -1, -1, -1, -1);
        case EK_OP_SELECT: return SEL(DOP_SEL_M_32, DOP_SEL_M_64, DOP_SEL_M_32, DOP_SEL_M_32, DOP_SEL_M_64, DOP_SEL_M_64);
        default: return -1;
    }
}

/* conversion src -> dst (cuda.h:236-247); mode = rounding for float->int */
int pick_cvt(ek_type src, ek_type dst) {
    Cls s = cls_of(src), d = cls_of(dst);
    if (s == C_BAD || d == C_BAD) return -1;
    static const int tab[6][6] = {
        /* from F32 */ { DOP_LOAD_32, DOP_CVT_F32_F64, DOP_CVT_F32_I32, DOP_CVT_F32_U32, DOP_CVT_F32_I64, DOP_CVT_F32_U64 },
        /* from F64 */ { DOP_CVT_F64_F32, DOP_LOAD_64, DOP_CVT_F64_I32, DOP_CVT_F64_U32, DOP_CVT_F64_I64, DOP_CVT_F64_U64 },
        /* from I32 */ { DOP_CVT_I32_F32, DOP_CVT_I32_F64, DOP_LOAD_32, DOP_LOAD_32, DOP_CVT_I32_I64, DOP_CVT_I32_I64 },
        /* from U32 */ { DOP_CVT_U32_F32, DOP_CVT_U32_F64, DOP_LOAD_32, DOP_LOAD_32, DOP_CVT_U32_U64, DOP_CVT_U32_U64 },
        /* from I64 */ { DOP_CVT_I64_F32, DOP_CVT_I64_F64, DOP_CVT_64_32, DOP_CVT_64_32, DOP_LOAD_64, DOP_LOAD_64 },
        /* from U64 */ { DOP_CVT_U64_F32, DOP_CVT_U64_F64, DOP_CVT_64_32, DOP_CVT_64_32, DOP_LOAD_64, DOP_LOAD_64 } };
    return tab[s][d];
}

int red_class(ek_type t) {
    switch (cls_of(t)) {
        case C_F32: return EK_RC_F32; case C_F64: return EK_RC_F64;
        case C_I32: return EK_RC_I32; case C_U32: return EK_RC_U32;
        case C_I64: return EK_RC_I64; default: return EK_RC_U64;
    }
}

uint64_t red_identity(int kind, int cls) {
    auto f32 = [](float f) { uint32_t u; memcpy(&u, &f, 4); return (uint64_t) u; };
    auto f64 = [](double f) { uint64_t u; memcpy(&u, &f, 8); return u; };
    switch (cls) {
        case EK_RC_F32: return kind == EK_RED_SUM ? f32(0.f) : kind == EK_RED_PROD ? f32(1.f) : kind == EK_RED_MIN ? 0x7f800000ull : 0xff800000ull;
        case EK_RC_F64: return kind == EK_RED_SUM ? f64(0.0) : kind == EK_RED_PROD ? f64(1.0) : kind == EK_RED_MIN ? 0x7ff0000000000000ull : 0xfff0000000000000ull;
        case EK_RC_I32: return kind == EK_RED_SUM ? 0 : kind == EK_RED_PROD ? 1 : kind == EK_RED_MIN ? 0x7fffffffull : 0x80000000ull;
        case EK_RC_U32: return kind == EK_RED_SUM ? 0 : kind == EK_RED_PROD ? 1 : kind == EK_RED_MIN ? 0xffffffffull : 0;
        case EK_RC_I64: return kind == EK_RED_SUM ? 0 : kind == EK_RED_PROD ? 1 : kind == EK_RED_MIN ? 0x7fffffffffffffffull : 0x8000000000000000ull;
        default:        return kind == EK_RED_SUM ? 0 : kind == EK_RED_PROD ? 1 : kind == EK_RED_MIN ? ~0ull : 0;
    }
}

/* ------------------------------------------------------------------ assembler */
/* operand positions of `op` that may be served from the accumulator (bit p = dep[p]) */
uint32_t acc_positions(const EkVariable &v) {
    ek_op op = v.op;
    if (op == EK_OP_LITERAL || op == EK_OP_INDEX) return 0;
    if (ek_op_unary(op)) return 1;
    if (ek_op_binary(op)) return 3;
    if (op == EK_OP_FMA || op == EK_OP_SELECT || op == EK_OP_FMA_NZ) return 7;
    if (ek_op_carlson3(op)) return 1;
    if (op == EK_OP_GATHER || op == EK_OP_SCATTER || op == EK_OP_SCATTER_ADD) return 2;   /* the index */
    if (op >= EK_OP_HSUM && op <= EK_OP_COUNT) return 1;
    return 0;
}

struct Assembler {
    EkContext &ctx;
    const Group &g;
    const std::unordered_set<uint32_t> &forced;
    Assembled out;

    std::unordered_map<uint32_t, Loc> loc;
    std::unordered_map<uint32_t, uint32_t> last_use;   /* var -> sched position of last consumer */
    std::unordered_map<uint32_t, uint32_t> epos;       /* var -> emit index */
    std::unordered_map<uint32_t, uint32_t> last_epos;  /* var -> max emit index among consumers */
    std::unordered_set<uint32_t> force_slot;           /* next consumer cannot take it from the accumulator */
    std::unordered_map<uint64_t, uint32_t> lit32, lit64;
    std::vector<uint8_t> slot_used;
    std::unordered_map<uint32_t, uint32_t> red_acc;    /* reduce var -> accumulator slot */
    std::unordered_set<uint32_t> direct;               /* wide inputs loaded with ld.global instead of TMA staging */
    std::unordered_set<uint32_t> implied_mask;         /* gathers / scatter_adds whose mask is implied by the range check of
                                                          their shared-memory table / bins (see mask_is_implied) */
    std::unordered_set<uint32_t> dead;                 /* mask variables that only fed such operations: not emitted */
    uint32_t acc_var = 0;
    uint32_t cur_e = 0;

    Assembler(EkContext &c, const Group &gr, const std::unordered_set<uint32_t> &f)
        : ctx(c), g(gr), forced(f) {}

    const EkVariable &var(uint32_t i) const { return ctx.vars[i]; }
    bool wide() const { return g.size > 1; }

    uint32_t lit_word(uint32_t w) {
        auto it = lit32.find(w);
        if (it != lit32.end()) return it->second;
        uint32_t idx = (uint32_t) out.lits.size();
        out.lits.push_back(w);
        lit32[w] = idx;
        return idx;
    }
    uint32_t lit_pair(uint64_t w) {
        auto it = lit64.find(w);
        if (it != lit64.end()) return it->second;
        uint32_t idx = (uint32_t) out.lits.size();
        out.lits.push_back((uint32_t) w); out.lits.push_back((uint32_t) (w >> 32));
        lit64[w] = idx;
        return idx;
    }
    /* argument words live after the literals; final uniform index = n_lit + argw (patched in finish) */
    uint32_t arg_ptr(uint32_t var_idx, bool output) {
        uint32_t idx = (uint32_t) out.argw.size();
        out.argw.push_back(0); out.argw.push_back(0);
        out.ptr_fix.push_back({ idx, var_idx, output });
        return idx;
    }

    uint32_t alloc_slots(uint32_t n) {
        for (uint32_t s = 0; s + n <= slot_used.size(); ++s) {
            bool ok = true;
            for (uint32_t k = 0; k < n; ++k) if (slot_used[s + k]) { ok = false; break; }
            if (ok) { for (uint32_t k = 0; k < n; ++k) slot_used[s + k] = 1; return s; }
        }
        uint32_t s = (uint32_t) slot_used.size();
        if (n == 2 && s > 0 && !slot_used[s - 1]) { slot_used[s - 1] = 1; slot_used.push_back(1); return s - 1; }
        for (uint32_t k = 0; k < n; ++k) slot_used.push_back(1);
        return s;
    }
    void free_slots(uint32_t s, uint32_t n) { for (uint32_t k = 0; k < n; ++k) slot_used[s + k] = 0; }

    /* uniform codes carry a marker that is rebased in finish():
       literal word i -> 0x8000 | i ; argument word j -> 0x8000 | 0x2000 | j ; scalar word -> 0x8000 | 0x1000 | k */
    static uint16_t uni_lit(uint32_t i) { return (uint16_t) (0x8000u | i); }
    static uint16_t uni_arg(uint32_t j) { return (uint16_t) (0x8000u | 0x2000u | j); }
    static uint16_t staged_code(uint32_t unit) { return (uint16_t) (EK_OPND_STAGED | unit); }

    bool fail(const std::string &m) { if (out.error.empty()) out.error = m; return false; }
    bool fail_resource(const std::string &m) { out.resource_error = true; return fail(m); }

    /* shared-memory operand code of a value that is NOT taken from the accumulator */
    uint16_t operand(uint32_t v) {
        auto it = loc.find(v);
        if (it == loc.end()) { fail("internal: operand " + std::to_string(v) + " has no location"); return EK_OPND_NONE; }
        switch (it->second.kind) {
            case Loc::UNI: return it->second.idx;
            case Loc::STAGED: return staged_code(it->second.idx);
            case Loc::SLOT: return it->second.idx;
            default: fail("internal: operand " + std::to_string(v) + " not materialised"); return EK_OPND_NONE;
        }
    }

    void release(uint32_t v, uint32_t pos) {
        auto it = last_use.find(v);
        if (it == last_use.end() || it->second != pos) return;
        auto l = loc.find(v);
        if (l != loc.end() && l->second.kind == Loc::SLOT) {
            free_slots(l->second.idx, ek_is_64(var(v).type) ? 2 : 1);
            l->second.kind = Loc::NONE;
        }
    }

    EkInstr mk(int op, uint32_t imm = 0) {
        EkInstr in;
        in.op = (uint16_t) op; in.flags = 0; in.dst = 0; in.b = EK_OPND_NONE; in.c = EK_OPND_NONE; in.a = EK_OPND_NONE; in.imm = imm;
        return in;
    }
    static void set_mark(EkInstr &in, uint32_t m) { in.flags = (uint16_t) ((in.flags & ~0x3000u) | (m << 12)); }
    void set_b(EkInstr &in, uint32_t v) { in.b = operand(v); in.flags |= EKF_HAS_B; if (ek_is_64(var(v).type)) in.flags |= EKF_B64; }
    void set_c(EkInstr &in, uint32_t v) { in.c = operand(v); in.flags |= EKF_HAS_C; if (ek_is_64(var(v).type)) in.flags |= EKF_C64; }
    void set_b_code(EkInstr &in, uint16_t code, bool is64) { in.b = code; in.flags |= EKF_HAS_B; if (is64) in.flags |= EKF_B64; }
    void set_c_code(EkInstr &in, uint16_t code, bool is64) { in.c = code; in.flags |= EKF_HAS_C; if (is64) in.flags |= EKF_C64; }

    /* make `v` the accumulator content: the load is fused into the next instruction (EKF_HAS_A) */
    uint32_t last_emitted_for = 0; /* variable whose value the last body instruction produced */
    uint32_t pending_a = 0;       /* variable to load into the accumulator by the next instruction */
    uint32_t pending_mod = 0;     /* EKF_NEG_A / EKF_ABS_A to apply to the accumulator input     */
    uint16_t pending_a_code = 0; bool pending_a_64 = false;
    void ensure_acc(uint32_t v) {
        if (acc_var == v) return;
        flush_pending();          /* (cannot stack two loads) */
        pending_a = v;
        pending_a_code = operand(v);      /* resolved now: the slot may be released before the push */
        pending_a_64 = ek_is_64(var(v).type);
        acc_var = v;
    }
    /* append an instruction to the body, attaching the pending accumulator load / modifiers */
    void push_body(EkInstr in) {
        if (pending_a) {
            in.a = pending_a_code;
            in.flags |= EKF_HAS_A;
            if (pending_a_64) in.flags |= EKF_A64;
            pending_a = 0;
        }
        in.flags |= (uint16_t) pending_mod;
        pending_mod = 0;
        out.body.push_back(in);
    }
    void flush_pending() {
        if (pending_a || pending_mod) push_body(mk(DOP_NOP));
    }

    /* give the value of `v` (just produced into the accumulator by `in`) a home */
    void place_result(EkInstr &in, uint32_t v) {
        const EkVariable &vv = var(v);
        bool is64 = ek_is_64(vv.type);
        auto le = last_epos.find(v);
        bool needs_slot = (le != last_epos.end() && le->second > cur_e + 1) || force_slot.count(v);
        if (needs_slot) {
            uint32_t s = alloc_slots(is64 ? 2 : 1);
            in.flags |= EKF_ST | (is64 ? EKF_R64 : 0); in.dst = (uint16_t) s;
            loc[v] = { Loc::SLOT, (uint16_t) s };
        } else {
            loc[v] = { Loc::PENDING, 0 };
        }
    }

    bool lit_emits(uint32_t idx) const {
        const EkVariable &v = var(idx);
        return v.op == EK_OP_LITERAL && v.size == g.size && ((v.ref_ext > 0 && !v.side_effect) || forced.count(idx));
    }
    bool boundary_input(uint32_t idx) const { return g.boundary.count(idx) != 0; }

    /* does this gather / scatter_add go through a table / privatised bins in shared memory? (the same tests as in
       emit_var) -- count = number of entries */
    bool uses_smem(const EkVariable &v, uint32_t &count) const {
        if (!wide() || v.extra_dep < EK_REG_RESERVED) return false;
        const EkVariable &pv = var(v.dep[0]), &tv = var(v.extra_dep);
        ek_type it = var(v.dep[1]).type;
        if (ek_is_64(it) || ek_is_signed(it) || tv.data != pv.data || ek_type_size(tv.type) != 4) return false;
        count = (uint32_t) tv.size;
        if (v.op == EK_OP_GATHER) {
            uint32_t stride = (uint32_t) (v.imm & 0x7fffu);
            return (stride == 0 || stride == 4) && ek_type_size(v.type) == 4 && !ek_is_64(v.type) && tv.size <= 4096;
        }
        if (v.op == EK_OP_SCATTER_ADD) {
            ek_type vt = var(v.dep[3]).type;
            uint32_t stride = (uint32_t) ((v.imm >> 32) & 0x7fffu);
            return ek_type_size(vt) == 4 && (stride == 0 || stride == 4) && tv.size <= 1024;
        }
        return false;
    }
    /* The shared-memory forms test `index < count` themselves.  A mask that is exactly `index < L` with a literal
       L >= count (the histogram idiom: idx < n_bins) adds nothing: the operation is given a literal-true mask, and if the
       comparison has no other use it is not computed at all (one dispatch and one slot less per tile). */
    bool mask_is_implied(const EkVariable &v) const {
        uint32_t count = 0;
        if ((v.op != EK_OP_GATHER && v.op != EK_OP_SCATTER_ADD) || !uses_smem(v, count)) return false;
        uint32_t m = v.dep[2];
        if (m < EK_REG_RESERVED) return false;
        const EkVariable &mv = var(m);
        if (mv.data != nullptr || mv.op != EK_OP_LT || mv.dep[0] != v.dep[1] || mv.size != v.size) return false;
        if (boundary_input(m)) return false;
        const EkVariable &lv = var(mv.dep[1]);
        if (lv.op != EK_OP_LITERAL || lv.data != nullptr || ek_is_64(lv.type) || ek_is_signed(var(mv.dep[0]).type) || ek_is_float(var(mv.dep[0]).type)) return false;
        return (uint32_t) lv.imm >= count;
    }

    /* a staged Float16 input whose one use is a conversion to Float32 is not unpacked into a slot up front: the
       conversion reads the staged tile itself (LD_U16 + CVT_F16_F32, one FOP_LD_F16 on the fast kernel) */
    bool f16_read_by_cvt(uint32_t idx) const {
        if (var(idx).type != EK_FLOAT16) return false;
        int uses = 0; bool cvt = false;
        for (uint32_t c : g.sched) {
            const EkVariable &cv = var(c);
            if (cv.data != nullptr || cv.direct_pointer || boundary_input(c) || cv.op == EK_OP_LITERAL || dead.count(c)) continue;
            for (int k = 0; k < 4; ++k)
                if (cv.dep[k] == idx) { ++uses; cvt = k == 0 && cv.op == EK_OP_CVT && cv.type == EK_FLOAT32; }
        }
        return uses == 1 && cvt;
    }

    bool run() {
        /* ---- pass 0: masks implied by the range check of a shared-memory table / bins ---- */
        {
            std::unordered_map<uint32_t, int> other_uses;
            for (uint32_t idx : g.sched) {
                const EkVariable &v = var(idx);
                if (v.data != nullptr || v.direct_pointer || boundary_input(idx) || v.op == EK_OP_LITERAL) continue;
                const bool implied = mask_is_implied(v);
                if (implied) implied_mask.insert(idx);
                for (int k = 0; k < 4; ++k) {
                    uint32_t d = v.dep[k];
                    if (d < EK_REG_RESERVED) continue;
                    if (!(implied && k == 2)) other_uses[d]++;
                }
            }
            for (uint32_t idx : implied_mask) {
                uint32_t m = var(idx).dep[2];
                const EkVariable &mv = var(m);
                if (other_uses[m] == 0 && mv.ref_ext == 0 && !mv.side_effect && !forced.count(m) && g.visited.count(m) &&
                    std::find(g.roots.begin(), g.roots.end(), m) == g.roots.end()) dead.insert(m);
            }
        }
        /* ---- pass 0b: wide inputs beyond the staging budget are loaded directly (ld.global) ---- */
        {
            uint32_t units = 0, count = 0;
            for (uint32_t idx : g.sched) {
                const EkVariable &v = var(idx);
                bool is_input = (v.data != nullptr && !v.direct_pointer) || boundary_input(idx);
                if (!is_input || v.size == 1 || !wide()) continue;
                uint32_t u = ek_type_size(v.type) == 8 ? 2 : 1;
                if (count >= EK_MAX_STAGED || units + u > EK_STAGE_UNIT_BUDGET) direct.insert(idx);
                else { units += u; ++count; }
            }
        }

        for (uint32_t idx : g.sched) {
            const EkVariable &v = var(idx);
            if (!v.direct_pointer && ek_is_64(v.type)) out.has64 = true;
        }

        /* ---- pass 1: emit indices, last uses, accumulator compatibility ---- */
        uint32_t e = 0;
        std::vector<uint32_t> emits(g.sched.size(), 0);
        uint32_t prev_emitted = 0;
        for (size_t i = 0; i < g.sched.size(); ++i) {
            uint32_t idx = g.sched[i];
            const EkVariable &v = var(idx);
            bool is_input = v.data != nullptr || v.direct_pointer || boundary_input(idx);
            bool emitting;
            if (is_input) emitting = direct.count(idx) != 0;
            else if (v.op == EK_OP_LITERAL) emitting = lit_emits(idx);
            else emitting = dead.count(idx) == 0;
            if (emitting) {
                ++e;
                bool computes = !is_input && v.op != EK_OP_LITERAL;
                if (computes) {
                    uint32_t accp = acc_positions(v);
                    bool prev_ok = false, prev_used = false;
                    for (int k = 0; k < 4; ++k) {
                        uint32_t d = v.dep[k];
                        if (d < EK_REG_RESERVED) continue;
                        if (k == 2 && implied_mask.count(idx)) continue;        /* (that operand is not read) */
                        last_use[d] = (uint32_t) i;
                        last_epos[d] = e;
                        if (d == prev_emitted) { prev_used = true; if (k < 3 && (accp >> k) & 1u) prev_ok = true; }
                    }
                    if (prev_used && !prev_ok) force_slot.insert(prev_emitted);
                }
                prev_emitted = idx;
            }
            emits[i] = e;
            epos[idx] = e;
        }

        /* ---- staged inputs / scalars / literals ---- */
        uint32_t unit = 0;
        std::vector<std::pair<uint32_t, size_t>> unpack;   /* (var, sched pos) */
        for (size_t i = 0; i < g.sched.size(); ++i) {
            uint32_t idx = g.sched[i];
            const EkVariable &v = var(idx);
            bool binput = boundary_input(idx);
            if (v.direct_pointer) {
                uint32_t a = arg_ptr(idx, false);
                loc[idx] = { Loc::UNI, uni_arg(a) };
            } else if (v.data != nullptr || binput) {
                size_t es = ek_type_size(v.type);
                if (v.size == 1 || !wide()) {
                    if (out.scalars.size() >= EK_MAX_SCALAR) return fail_resource("too many scalar inputs in one kernel (limit " + std::to_string(EK_MAX_SCALAR) + ")");
                    uint32_t sidx = (uint32_t) out.scalars.size();
                    out.scalars.push_back({ idx });
                    loc[idx] = { Loc::UNI, (uint16_t) (0x8000u | 0x1000u | (2u * sidx)) };   /* rebased in finish */
                } else if (direct.count(idx)) {
                    if (v.size != g.size) return fail("encountered arrays of incompatible size");
                    out.bytes_in += (uint64_t) v.size * es;       /* emitted as LDG in pass 2 */
                } else {
                    if (v.size != g.size) return fail("encountered arrays of incompatible size");
                    uint32_t units = es == 8 ? 2 : 1;
                    out.staged.push_back({ idx, (uint16_t) unit, (uint8_t) es });
                    loc[idx] = { Loc::STAGED, (uint16_t) unit };
                    if (es != 4 && !f16_read_by_cvt(idx)) unpack.push_back({ idx, i });
                    unit += units;
                    out.bytes_in += (uint64_t) v.size * es;
                }
            } else if (v.op == EK_OP_LITERAL) {
                if (ek_is_64(v.type)) loc[idx] = { Loc::UNI, uni_lit(lit_pair(v.imm)) };
                else loc[idx] = { Loc::UNI, uni_lit(lit_word(register_word(v.type, v.imm))) };
            }
        }
        out.n_in_units = unit;

        /* ---- reduction accumulators persist across tiles: reserve their slots up front ---- */
        for (uint32_t idx : g.sched) {
            const EkVariable &v = var(idx);
            if (v.data != nullptr || boundary_input(idx) || !is_reduce(v.op)) continue;
            bool w64 = ek_is_64(var(v.dep[0]).type) && v.op != EK_OP_ALL && v.op != EK_OP_ANY && v.op != EK_OP_COUNT;
            red_acc[idx] = alloc_slots(w64 ? 2 : 1);
        }

        /* ---- body prologue: unpack non-32-bit staged inputs into slots ---- */
        for (auto &u : unpack) {
            uint32_t idx = u.first;
            const EkVariable &v = var(idx);
            int op;
            switch (v.type) {
                case EK_BOOL: case EK_UINT8: op = DOP_LD_U8; break;
                case EK_INT8: op = DOP_LD_S8; break;
                case EK_UINT16: case EK_FLOAT16: op = DOP_LD_U16; break;
                case EK_INT16: op = DOP_LD_S16; break;
                default: op = DOP_LD_64; break;
            }
            EkInstr in = mk(op);
            in.b = staged_code(loc[idx].idx);       /* raw staged code; no generic fetch (EKF_HAS_B clear) */
            bool is64 = ek_is_64(v.type);
            uint32_t s = alloc_slots(is64 ? 2 : 1);
            in.flags |= EKF_ST | (is64 ? EKF_R64 : 0); in.dst = (uint16_t) s;
            loc[idx] = { Loc::SLOT, (uint16_t) s };
            out.body.push_back(in);
            if (last_use.find(idx) == last_use.end()) free_slots(s, is64 ? 2 : 1);
        }
        acc_var = 0;

        /* ---- pass 2: emit ---- */
        for (size_t i = 0; i < g.sched.size(); ++i) {
            uint32_t idx = g.sched[i];
            const EkVariable &v = var(idx);
            if (direct.count(idx)) {
                cur_e = emits[i];
                int op;
                switch (v.type) {
                    case EK_BOOL: case EK_UINT8: op = DOP_LDG_U8; break;
                    case EK_INT8: op = DOP_LDG_S8; break;
                    case EK_UINT16: case EK_FLOAT16: op = DOP_LDG_U16; break;
                    case EK_INT16: op = DOP_LDG_S16; break;
                    case EK_INT32: case EK_UINT32: case EK_FLOAT32: op = DOP_LDG_32; break;
                    default: op = DOP_LDG_64; break;
                }
                uint32_t pa = arg_ptr(idx, false);
                EkInstr in = mk(op, uni_arg(pa) & 0x7fffu);
                set_mark(in, 1);               /* marker: imm holds an argument-word index to rebase */
                flush_pending();
                place_result(in, idx);
                push_body(in);
                acc_var = idx;
                continue;
            }
            if (v.data != nullptr || v.direct_pointer || boundary_input(idx)) continue;
            if (v.op == EK_OP_LITERAL && !lit_emits(idx)) continue;
            if (dead.count(idx)) continue;
            cur_e = emits[i];
            if (!emit_var(idx, (uint32_t) i)) return false;
        }
        flush_pending();
        return finish();
    }

    bool emit_var(uint32_t idx, uint32_t pos) {
        const EkVariable &v = var(idx);
        ek_op op = v.op;
        ek_type t = v.type;
        bool is64 = ek_is_64(t);
        out.n_arith++;
        uint32_t d0 = v.dep[0], d1 = v.dep[1], d2 = v.dep[2], d3 = v.dep[3];

        auto after = [&]() { if (d0) release(d0, pos); if (d1) release(d1, pos); if (d2) release(d2, pos); if (d3) release(d3, pos); };
        /* Float16 is a storage format (DESIGN.md §4): literals, conversions (incl. floor2int / ceil2int), bit casts,
           select, gather and scatter move or convert its bits; everything else converts to Float32 first, as the
           reference's half does */
        if (op != EK_OP_LITERAL && op != EK_OP_MOV && op != EK_OP_CVT && op != EK_OP_FLOOR2INT && op != EK_OP_CEIL2INT &&
            op != EK_OP_BITCAST && op != EK_OP_SELECT && op != EK_OP_GATHER && op != EK_OP_SCATTER) {
            bool f16 = t == EK_FLOAT16;
            for (int k = 0; k < 4; ++k) if (v.dep[k] >= EK_REG_RESERVED && var(v.dep[k]).type == EK_FLOAT16) f16 = true;
            if (f16) return fail(std::string("op ") + ek_op_name(op) + " is not supported on Float16, a storage format: convert to Float32 to compute");
        }

        /* ---------------- reductions ---------------- */
        if (is_reduce(op)) {
            ek_type xt = var(d0).type;
            int kind, cls = red_class(xt);
            switch (op) {
                case EK_OP_HSUM: kind = EK_RED_SUM; break;
                case EK_OP_HPROD: kind = EK_RED_PROD; break;
                case EK_OP_HMAX: kind = EK_RED_MAX; break;
                case EK_OP_HMIN: kind = EK_RED_MIN; break;
                case EK_OP_ALL: kind = EK_RED_MIN; cls = EK_RC_U32; break;
                case EK_OP_ANY: kind = EK_RED_MAX; cls = EK_RC_U32; break;
                default: kind = EK_RED_SUM; cls = EK_RC_U32; break;   /* COUNT */
            }
            if (out.n_red >= EK_MAX_RED) return fail_resource("too many reductions in one kernel");
            bool w64 = cls >= EK_RC_F64;
            uint32_t ridx = out.n_red++;
            uint32_t acc = red_acc[idx];                 /* reserved in run(); never freed */
            uint64_t ident = red_identity(kind, cls);
            EkInstr ini = mk(w64 ? DOP_LOAD_64 : DOP_LOAD_32);
            set_b_code(ini, w64 ? uni_lit(lit_pair(ident)) : uni_lit(lit_word((uint32_t) ident)), w64);
            ini.flags |= EKF_ST | (w64 ? EKF_R64 : 0); ini.dst = (uint16_t) acc;
            out.init.push_back(ini);
            EkInstr *last = out.body.empty() ? nullptr : &out.body.back();
            const bool mask_red = op == EK_OP_ALL || op == EK_OP_ANY || op == EK_OP_COUNT;
            if (mask_red) {
                /* a borrowed mask may hold any non-zero byte for `true` (2, 0xff): fold (x != 0), so that COUNT adds 1
                   per true element and ALL / ANY produce a canonical 0 / 1 */
                ensure_acc(d0);
                push_body(mk(DOP_NEZ_32));
                acc_var = 0;
                EkInstr in = mk(DOP_RACC, (uint32_t) kind | ((uint32_t) cls << 8));
                in.dst = (uint16_t) acc;
                push_body(in);
                last_emitted_for = 0;
            } else if (acc_var == d0 && !pending_a && !pending_mod && last && last_emitted_for == d0 &&
                !(last->flags & (EKF_ST | EKF_HAS_A | EKF_RACC))) {
                /* fused into the instruction that produces the value */
                last->flags |= EKF_RACC;
                last->dst = (uint16_t) acc;
                last->a = (uint16_t) ((uint32_t) kind | ((uint32_t) cls << 8));
            } else {
                ensure_acc(d0);
                EkInstr in = mk(DOP_RACC, (uint32_t) kind | ((uint32_t) cls << 8));
                in.dst = (uint16_t) acc;
                push_body(in);
                last_emitted_for = 0;        /* the last instruction is no longer the producer of d0 */
            }
            uint32_t pa = arg_ptr(idx, true);
            out.outputs.push_back({ idx, pa, 8 });
            EkInstr fi = mk(DOP_RFIN, (uint32_t) kind | ((uint32_t) cls << 8) | (ridx << 16));
            set_b_code(fi, (uint16_t) acc, w64);
            fi.dst = (uint16_t) pa; set_mark(fi, 2);     /* marker: dst holds an argument-word index to rebase */
            out.fini.push_back(fi);
            after();
            return out.error.empty();
        }

        EkInstr in = mk(DOP_NOP);
        bool produces = true;

        /* operand that is currently in the accumulator among the positions the op accepts */
        auto acc_at = [&](uint32_t a, uint32_t b, uint32_t c) -> int {
            if (a && a == acc_var) return 0;
            if (b && b == acc_var) return 1;
            if (c && c == acc_var) return 2;
            return -1;
        };
        /* fetch operand v into B / C, or alias the accumulator when it is the same value */
        auto put_b = [&](EkInstr &ins, uint32_t vv) { if (vv == acc_var) { ensure_slot_or_alias(ins, vv, true); } else set_b(ins, vv); };
        auto put_c = [&](EkInstr &ins, uint32_t vv) { if (vv == acc_var) { ensure_slot_or_alias(ins, vv, false); } else set_c(ins, vv); };

        switch (op) {
            case EK_OP_INDEX:
                in = mk(DOP_INDEX);
                break;
            case EK_OP_LITERAL:
                in = mk(is64 ? DOP_LOAD_64 : DOP_LOAD_32);
                set_b_code(in, loc[idx].idx, is64);
                break;
            case EK_OP_CVT: case EK_OP_FLOOR2INT: case EK_OP_CEIL2INT: {
                ek_type st = var(d0).type;
                int dop;
                /* Float16 converts through Float32 (half(x) = float32_to_float16(float(x)), Value(h) = Value(float(h)) in the
                   reference): `first` is the leg to or from Float32 that runs before `dop` */
                int first = -1;
                if (t == EK_BOOL && st != EK_BOOL) {
                    if (ek_is_float(st) || ek_is_64(st)) return fail("conversion to bool from this type is not supported");
                    dop = DOP_NEZ_32;
                } else if (st == EK_FLOAT16 && t != EK_FLOAT16) {
                    first = DOP_CVT_F16_F32;
                    dop = pick_cvt(EK_FLOAT32, t);
                } else if (t == EK_FLOAT16 && st != EK_FLOAT16) {
                    first = st == EK_FLOAT32 ? -1 : pick_cvt(st, EK_FLOAT32);
                    dop = DOP_CVT_F32_F16;
                } else dop = pick_cvt(st, t);
                if (dop < 0) return fail("unsupported conversion");
                uint32_t mode = op == EK_OP_FLOOR2INT ? EK_RM : op == EK_OP_CEIL2INT ? EK_RP : EK_RZ;
                if (st == EK_FLOAT16 && loc[d0].kind == Loc::STAGED) {
                    /* (f16_read_by_cvt: the staged tile is read here) */
                    flush_pending();
                    EkInstr ld = mk(DOP_LD_U16);
                    ld.b = staged_code(loc[d0].idx);
                    push_body(ld);
                    acc_var = d0;
                } else ensure_acc(d0);
                if (first >= 0 && dop == DOP_LOAD_32) { dop = first; first = -1; }     /* Float16 -> Float32: one instruction */
                if (first >= 0) push_body(mk(first));
                in = mk(dop == DOP_LOAD_32 || dop == DOP_LOAD_64 ? DOP_NOP : dop, mode);
            } break;
            case EK_OP_BITCAST: {
                if (ek_type_size(var(d0).type) != ek_type_size(t)) return fail("bitcast between types of different size");
                ensure_acc(d0);
                in = mk(DOP_NOP);
            } break;
            case EK_OP_GATHER: {
                const EkVariable &pv = var(d0);
                uint32_t stride = (uint32_t) (v.imm & 0x7fffu);
                if (stride == 0) stride = (uint32_t) ek_type_size(t);
                ek_type it = var(d1).type;
                bool sgn = ek_is_signed(it);
                int dop;
                bool smem_table = false;
                switch (t) {
                    case EK_BOOL: case EK_UINT8: dop = DOP_GATHER_U8; break;
                    case EK_INT8: dop = DOP_GATHER_S8; break;
                    case EK_UINT16: case EK_FLOAT16: dop = DOP_GATHER_U16; break;
                    case EK_INT16: dop = DOP_GATHER_S16; break;
                    case EK_INT32: case EK_UINT32: case EK_FLOAT32: dop = DOP_GATHER_32; break;
                    default: dop = DOP_GATHER_64; break;
                }
                /* small 32-bit tables are staged in shared memory once per CTA */
                if (dop == DOP_GATHER_32 && stride == 4 && v.extra_dep >= EK_REG_RESERVED && wide() && !ek_is_64(it) && !sgn) {
                    const EkVariable &tv = var(v.extra_dep);
                    if (tv.data == pv.data && tv.size <= 4096 && ek_type_size(tv.type) == 4) smem_table = true;
                }
                uint32_t pa = loc[d0].idx;   /* uniform code of the pointer words */
                ensure_acc(d1);
                if (smem_table) {
                    uint32_t count = (uint32_t) var(v.extra_dep).size;
                    uint32_t di = (uint32_t) out.argw.size();
                    out.argw.push_back(out.extra_bytes); out.argw.push_back(count); out.argw.push_back(1); out.argw.push_back(pa);
                    out.extra_bytes += (count * 4 + 15) & ~15u;
                    out.extra_items.push_back({ di, count, 0 });
                    EkInstr li = mk(DOP_SMEM_LOAD_TABLE, di); set_mark(li, 1);
                    out.init.push_back(li);
                    in = mk(DOP_GATHER_32_SMEM, di); set_mark(in, 1);
                } else {
                    in = mk(dop, (sgn ? 0x80000000u : 0u) | (stride << 16) | pa);
                    set_mark(in, 3);         /* marker: imm low 16 bits hold a uniform code to rebase */
                }
                if (implied_mask.count(idx)) {
                    if (!smem_table) return fail("internal: implied mask on a gather without a shared-memory table");
                    set_b_code(in, uni_lit(lit_word(1u)), false);
                } else put_b(in, d2);
                if (ek_is_64(it)) in.flags |= EKF_A64;
            } break;
            case EK_OP_SCATTER: case EK_OP_SCATTER_ADD: {
                const EkVariable &pv = var(d0);
                ek_type vt = var(d3).type;
                uint32_t stride = (uint32_t) ((v.imm >> 32) & 0x7fffu);
                if (stride == 0) stride = (uint32_t) ek_type_size(vt);
                ek_type it = var(d1).type;
                bool sgn = ek_is_signed(it);
                int dop; bool smem_bins = false;
                size_t es = ek_type_size(vt);
                if (op == EK_OP_SCATTER) {
                    dop = es == 1 ? DOP_SCATTER_8 : es == 2 ? DOP_SCATTER_16 : es == 4 ? DOP_SCATTER_32 : DOP_SCATTER_64;
                } else {
                    switch (vt) {
                        case EK_FLOAT32: dop = DOP_SCATTER_ADD_F32; break;
                        case EK_INT32: case EK_UINT32: dop = DOP_SCATTER_ADD_I32; break;
                        case EK_FLOAT64: dop = DOP_SCATTER_ADD_F64; break;
                        case EK_INT64: case EK_UINT64: dop = DOP_SCATTER_ADD_I64; break;
                        default: return fail("scatter_add: unsupported type");
                    }
                    if (es == 4 && stride == 4 && v.extra_dep >= EK_REG_RESERVED && wide() && !ek_is_64(it) && !sgn) {
                        const EkVariable &tv = var(v.extra_dep);
                        if (tv.data == pv.data && tv.size <= 1024 && ek_type_size(tv.type) == 4) smem_bins = true;
                    }
                }
                uint32_t pa = loc[d0].idx;
                ensure_acc(d1);
                if (smem_bins) {
                    uint32_t count = (uint32_t) var(v.extra_dep).size;
                    /* integer bins: up to 32 copies shared by (warp, lane & 3), native shared-memory atomics (ATOMS.ADD).
                       float bins: a shared-memory float atomicAdd is a compare-and-swap loop (ATOMS.CAST.SPIN) that
                       crawls under contention, so small float targets get one private copy per thread instead
                       (plain read-modify-write, bank = thread id, no atomics) */
                    uint32_t copies = (dop == DOP_SCATTER_ADD_F32 && count <= 32u) ? 256u : std::max(1u, std::min(32u, 4096u / count));
                    uint32_t di = (uint32_t) out.argw.size();
                    out.argw.push_back(out.extra_bytes); out.argw.push_back(count); out.argw.push_back(copies); out.argw.push_back(pa);
                    out.extra_bytes += (count * copies * 4 + 15) & ~15u;
                    out.extra_items.push_back({ di, count, (uint8_t) (dop == DOP_SCATTER_ADD_F32 ? 1 : 2) });
                    /* float bins start at -0.0, not +0.0: x + -0.0 == x for every x, so a bin that receives nothing (or
                       only -0.0) leaves a -0.0 target element as it is, and the flush skips exactly those bins */
                    EkInstr zi = mk(DOP_SMEM_ZERO, di); set_mark(zi, 1);
                    zi.dst = dop == DOP_SCATTER_ADD_F32 ? 1 : 0;
                    out.init.push_back(zi);
                    EkInstr fl = mk(dop == DOP_SCATTER_ADD_F32 ? DOP_SMEM_FLUSH_ADD_F32 : DOP_SMEM_FLUSH_ADD_I32, di); set_mark(fl, 1);
                    out.fini.push_back(fl);
                    in = mk(dop == DOP_SCATTER_ADD_F32 ? DOP_SCATTER_ADD_F32_SMEM : DOP_SCATTER_ADD_I32_SMEM, di); set_mark(in, 1);
                } else {
                    in = mk(dop, (sgn ? 0x80000000u : 0u) | (stride << 16) | pa);
                    set_mark(in, 3);
                }
                put_b(in, d3);
                if (implied_mask.count(idx)) {
                    if (!smem_bins) return fail("internal: implied mask on a scatter_add without privatised bins");
                    set_c_code(in, uni_lit(lit_word(1u)), false);
                } else put_c(in, d2);
                if (ek_is_64(it)) in.flags |= EKF_A64;
                produces = false;
            } break;
            case EK_OP_SELECT: {
                int p = acc_at(d0, d1, d2);
                if (p < 0) { ensure_acc(d0); p = 0; }
                int dop = p == 0 ? (is64 ? DOP_SEL_M_64 : DOP_SEL_M_32) : p == 1 ? (is64 ? DOP_SEL_T_64 : DOP_SEL_T_32)
                                                                                 : (is64 ? DOP_SEL_F_64 : DOP_SEL_F_32);
                in = mk(dop);
                if (p == 0) { put_b(in, d1); put_c(in, d2); }
                else if (p == 1) { put_b(in, d0); put_c(in, d2); }
                else { put_b(in, d0); put_c(in, d1); }
            } break;
            case EK_OP_FMA: case EK_OP_FMA_NZ: {
                int p = acc_at(d0, d1, d2);
                if (p < 0) { ensure_acc(d0); p = 0; }
                Cls c = cls_of(t);
                int base, basec;
                if (op == EK_OP_FMA) {
                    base = SEL(DOP_FMA_F32, DOP_FMA_F64, DOP_MAD_I32, DOP_MAD_I32, DOP_MAD_I64, DOP_MAD_I64);
                    basec = SEL(DOP_FMAC_F32, DOP_FMAC_F64, DOP_MADC_I32, DOP_MADC_I32, DOP_MADC_I64, DOP_MADC_I64);
                } else {
                    if (c != C_F32 && c != C_F64) return fail("fma_nz: floating point only");
                    base = c == C_F32 ? DOP_FMANZ_F32 : DOP_FMANZ_F64;
                    basec = c == C_F32 ? DOP_FMANZC_F32 : DOP_FMANZC_F64;
                }
                in = mk(p == 2 ? basec : base);
                if (p == 0) { put_b(in, d1); put_c(in, d2); }
                else if (p == 1) { put_b(in, d0); put_c(in, d2); }
                else { put_b(in, d0); put_c(in, d1); }
            } break;
            case EK_OP_CARLSON_RF: case EK_OP_CARLSON_RD: {
                /* x is the accumulator (acc_positions): when it holds y or z, x is loaded by the instruction itself */
                int dop = pick_op(op, t, var(d0).type);
                if (dop < 0) return fail(std::string("op ") + ek_op_name(op) + " not supported for type " + ek_type_name(t));
                ensure_acc(d0);
                in = mk(dop);
                put_b(in, d1); put_c(in, d2);
            } break;
            case EK_OP_AND: case EK_OP_OR: {
                ek_type bt = var(d1).type;
                if (t != EK_BOOL && bt == EK_BOOL) {
                    /* value & mask = select(mask, value, 0); value | mask = select(mask, ~0, value) (cuda.h:545-572), ~0 as the
                       type's register holds it (0xff for UInt8) */
                    uint16_t k = is64 ? uni_lit(lit_pair(op == EK_OP_AND ? 0ull : ~0ull))
                                      : uni_lit(lit_word(op == EK_OP_AND ? 0u : register_word(t, ~0ull)));
                    int p = acc_at(d0, d1, 0);
                    if (p < 0) { ensure_acc(d0); p = 0; }
                    if (op == EK_OP_AND) {
                        if (p == 0) { in = mk(is64 ? DOP_SEL_T_64 : DOP_SEL_T_32); put_b(in, d1); set_c_code(in, k, is64); }
                        else        { in = mk(is64 ? DOP_SEL_M_64 : DOP_SEL_M_32); put_b(in, d0); set_c_code(in, k, is64); }
                    } else {
                        if (p == 0) { in = mk(is64 ? DOP_SEL_F_64 : DOP_SEL_F_32); put_b(in, d1); set_c_code(in, k, is64); }
                        else        { in = mk(is64 ? DOP_SEL_M_64 : DOP_SEL_M_32); set_b_code(in, k, is64); put_c(in, d0); }
                    }
                    break;
                }
            }   /* fall through */
            default: {
                if (ek_op_unary(op)) {                                    /* unary */
                    ek_type at = var(d0).type;
                    int dop = pick_op(op, t, at);
                    if (dop < 0) return fail(std::string("op ") + ek_op_name(op) + " not supported for type " + ek_type_name(t));
                    ensure_acc(d0);
                    in = mk(dop == DOP_LOAD_32 || dop == DOP_LOAD_64 ? DOP_NOP : dop);
                } else if (ek_op_binary(op)) {                            /* binary */
                    ek_type at = var(d0).type;
                    int p = acc_at(d0, d1, 0);
                    if (p < 0) { ensure_acc(d0); p = 0; }
                    ek_op eop = op;
                    bool reversed = false;
                    if (p == 1) {
                        switch (op) {
                            case EK_OP_GT: eop = EK_OP_LT; break;
                            case EK_OP_GE: eop = EK_OP_LE; break;
                            case EK_OP_LT: eop = EK_OP_GT; break;
                            case EK_OP_LE: eop = EK_OP_GE; break;
                            case EK_OP_SUB: case EK_OP_DIV: case EK_OP_MOD: case EK_OP_SHL: case EK_OP_SHR: case EK_OP_ATAN2:
                            case EK_OP_POW: case EK_OP_HYPOT: case EK_OP_CARLSON_RC: reversed = true; break;
                            case EK_OP_MIN: case EK_OP_MAX: reversed = ek_is_float(t); break;
                            default: break;       /* commutative */
                        }
                    }
                    int dop = pick_op(eop, t, at);
                    if (dop < 0) return fail(std::string("op ") + ek_op_name(op) + " not supported for type " + ek_type_name(op >= EK_OP_GT && op <= EK_OP_NE ? at : t));
                    if (reversed) { dop = reversed_op(dop); if (dop < 0) return fail("internal: no reversed variant"); }
                    in = mk(dop);
                    put_b(in, p == 0 ? d1 : d0);
                    /* 64-bit shifts take a 32-bit count (cuda.h:503-505): only the low plane of the count is read */
                    if ((op == EK_OP_SHL || op == EK_OP_SHR) && is64 && !reversed) in.flags &= ~EKF_B64;
                } else return fail(std::string("unsupported op ") + ek_op_name(op));
            } break;
        }

        int nop = -1;
        bool arith_narrow = (op >= EK_OP_NEG && op <= EK_OP_ABS) || (op >= EK_OP_ADD && op <= EK_OP_SHR) ||
                            op == EK_OP_FMA || op == EK_OP_NOT || op == EK_OP_CVT || op == EK_OP_FLOOR2INT || op == EK_OP_CEIL2INT;
        if (arith_narrow) nop = norm_op(t);
        /* Float16 bits are held zero-extended, Int16 sign-extended: a bit cast between the two re-extends */
        if (op == EK_OP_BITCAST && t == EK_FLOAT16 && var(d0).type == EK_INT16) nop = DOP_ZEXT16;
        if (op == EK_OP_BITCAST && t == EK_INT16 && var(d0).type == EK_FLOAT16) nop = DOP_SEXT16;

        bool fused_mod = false;
        if (nop >= 0 && produces) {
            push_body(in);
            EkInstr nn = mk(nop);
            after();
            place_result(nn, idx);
            push_body(nn);
            acc_var = idx;
        } else {
            after();
            if (produces) place_result(in, idx);
            bool will_store = produces && ((!v.side_effect && v.ref_ext > 0 && v.size == g.size) || forced.count(idx));
            if ((in.op == DOP_NEG_F32 || in.op == DOP_ABS_F32) && !(in.flags & EKF_ST) && !will_store && !pending_mod &&
                single_acc_consumer(idx)) {
                /* fold -x / |x| into the consumer as an accumulator input modifier */
                pending_mod = in.op == DOP_NEG_F32 ? EKF_NEG_A : EKF_ABS_A;
                fused_mod = true;
            } else if (!(in.op == DOP_NOP && !(in.flags & EKF_ST) && !pending_a && !pending_mod)) {
                /* (a pure rename that needs no slot and carries no pending load emits nothing) */
                push_body(in);
            }
            if (produces) acc_var = idx;
        }
        last_emitted_for = (!fused_mod && produces && !out.body.empty()) ? idx : 0;

        /* ---- output store (jit.cu:1165-1205) ---- */
        if (produces) {
            bool store = (!v.side_effect && v.ref_ext > 0 && v.size == g.size) || forced.count(idx);
            if (store) {
                size_t es = ek_type_size(t);
                uint32_t pa = arg_ptr(idx, true);
                out.outputs.push_back({ idx, pa, std::max<size_t>(v.size * es, 8) });
                int sop = es == 1 ? DOP_ST_8 : es == 2 ? DOP_ST_16 : es == 4 ? DOP_ST_32 : DOP_ST_64;
                flush_pending();
                EkInstr *last = out.body.empty() ? nullptr : &out.body.back();
                if (es == 4 && last && imm_free(last->op) && !(last->flags & (EKF_STG | 0x3000u)) && last_emitted_for == idx) {
                    last->flags |= EKF_STG;            /* fused into the producing instruction */
                    last->imm = pa; set_mark(*last, 1);
                } else {
                    EkInstr st = mk(sop, pa);
                    set_mark(st, 1);
                    push_body(st);
                }
                out.bytes_out += (uint64_t) v.size * es;
            }
        }
        return out.error.empty();
    }

    /* the value in the accumulator is also needed as B / C of the same instruction (e.g. t*t):
       it must have a slot (guaranteed by force_slot in pass 1 when last use > e+1) -- otherwise spill
       it to a scratch slot first */
    void ensure_slot_or_alias(EkInstr &ins, uint32_t vv, bool as_b) {
        auto l = loc.find(vv);
        bool resident = l != loc.end() && (l->second.kind == Loc::SLOT || l->second.kind == Loc::STAGED || l->second.kind == Loc::UNI);
        if (!resident) {
            bool is64 = ek_is_64(var(vv).type);
            uint32_t s = alloc_slots(is64 ? 2 : 1);
            EkInstr sp = mk(DOP_NOP);
            sp.flags |= EKF_ST | (is64 ? EKF_R64 : 0); sp.dst = (uint16_t) s;
            push_body(sp);
            loc[vv] = { Loc::SLOT, (uint16_t) s };
            scratch.push_back({ s, is64 ? 2u : 1u });
        }
        if (as_b) set_b(ins, vv); else set_c(ins, vv);
    }
    std::vector<std::pair<uint32_t, uint32_t>> scratch;

    /* does the instruction leave its imm field unused (so that EKF_STG can use it)? */
    static bool imm_free(int op) {
        if (ek_dop_ext(op)) return true;
        if (op >= DOP_CVT_F32_I32 && op <= DOP_CVT_64_32) return false;
        if (op >= DOP_LD_U8) return false;          /* loads, stores, gathers, scatters, reductions, smem helpers */
        return true;
    }
    /* v is consumed exactly once, by the next emitted instruction, through the accumulator */
    bool single_acc_consumer(uint32_t vidx) {
        auto le = last_epos.find(vidx);
        if (le == last_epos.end() || le->second != cur_e + 1 || force_slot.count(vidx)) return false;
        /* find the consumer and make sure v appears once among its operands */
        for (size_t i = 0; i < g.sched.size(); ++i) {
            auto ep = epos.find(g.sched[i]);
            if (ep == epos.end() || ep->second != cur_e + 1) continue;
            const EkVariable &c = var(g.sched[i]);
            if (c.data != nullptr || c.op == EK_OP_LITERAL) continue;
            int cnt = 0;
            for (int k = 0; k < 4; ++k) if (c.dep[k] == vidx) ++cnt;
            return cnt == 1;
        }
        return false;
    }

    static int reversed_op(int dop) {
        switch (dop) {
            case DOP_SUB_F32: return DOP_SUBR_F32; case DOP_DIV_F32: return DOP_DIVR_F32; case DOP_ATAN2_F32: return DOP_ATAN2R_F32;
            case DOP_POW_F32: return DOP_POWR_F32; case DOP_HYPOT_F32: return DOP_HYPOTR_F32;
            case DOP_CARLSON_RC_F32: return DOP_CARLSON_RCR_F32;
            case DOP_MIN_F32: return DOP_MINR_F32; case DOP_MAX_F32: return DOP_MAXR_F32;
            case DOP_SUB_F64: return DOP_SUBR_F64; case DOP_DIV_F64: return DOP_DIVR_F64;
            case DOP_MIN_F64: return DOP_MINR_F64; case DOP_MAX_F64: return DOP_MAXR_F64;
            case DOP_SUB_I32: return DOP_SUBR_I32; case DOP_DIV_I32: return DOP_DIVR_I32; case DOP_DIV_U32: return DOP_DIVR_U32;
            case DOP_MOD_I32: return DOP_MODR_I32; case DOP_MOD_U32: return DOP_MODR_U32;
            case DOP_SHL_32: return DOP_SHLR_32; case DOP_SHR_I32: return DOP_SHRR_I32; case DOP_SHR_U32: return DOP_SHRR_U32;
            case DOP_SUB_I64: return DOP_SUBR_I64; case DOP_DIV_I64: return DOP_DIVR_I64; case DOP_DIV_U64: return DOP_DIVR_U64;
            case DOP_MOD_I64: return DOP_MODR_I64; case DOP_MOD_U64: return DOP_MODR_U64;
            case DOP_SHL_64: return DOP_SHLR_64; case DOP_SHR_I64: return DOP_SHRR_I64; case DOP_SHR_U64: return DOP_SHRR_U64;
            default: return -1;
        }
    }

    /* Early release (single-buffered staging): find the body instruction after which most staged bytes are
       dead while most of the tile's work is still ahead; the kernel starts streaming those inputs for the
       CTA's next tile right there. */
    void plan_release() {
        size_t ns = out.staged.size(), nb = out.body.size();
        if (ns == 0 || ns > 16 || nb < 3) return;
        /* programs with gathers / scatters are bound by those, not by streaming their inputs: there the release's
           barrier and extra dispatch cost more than the overlap gains (C3 measured 3-7 % slower with it on an H100) */
        for (const EkInstr &in : out.body) if (in.op >= DOP_GATHER_32 && in.op <= DOP_SCATTER_ADD_I32_SMEM) return;
        std::vector<int> last(ns, -1);
        auto unit_of = [&](uint16_t code) -> int { return (code != EK_OPND_NONE && !(code & 0x8000u) && (code & EK_OPND_STAGED)) ? (int) (code & 0x3fffu) : -1; };
        for (size_t i = 0; i < nb; ++i) {
            const EkInstr &in = out.body[i];
            int u[3] = { (in.flags & EKF_HAS_A) ? unit_of(in.a) : -1,
                         ((in.flags & EKF_HAS_B) || (in.op >= DOP_LD_U8 && in.op <= DOP_LD_64)) ? unit_of(in.b) : -1,
                         (in.flags & EKF_HAS_C) ? unit_of(in.c) : -1 };
            for (int q = 0; q < 3; ++q) {
                if (u[q] < 0) continue;
                for (size_t k = 0; k < ns; ++k) if (out.staged[k].unit == u[q]) last[k] = (int) i;
            }
        }
        double best = 0; int best_i = -1; uint32_t best_mask = 0;
        size_t total_bytes = 0;
        for (size_t k = 0; k < ns; ++k) total_bytes += out.staged[k].esize;
        /* heavier instructions weigh more: transcendental ~ 8, others 1 */
        auto weight = [&](const EkInstr &in) -> double {
            switch (in.op) { case DOP_SIN_F32: case DOP_COS_F32: case DOP_EXP_F32: case DOP_LOG_F32: return 8.0;
                             case DOP_TAN_F32: case DOP_COT_F32: return 12.0;
                             case DOP_ASIN_F32: case DOP_ACOS_F32: case DOP_ATAN_F32: case DOP_ATAN2_F32: case DOP_ATAN2R_F32: return 10.0;
                             case DOP_COSH_F32: return 10.0;
                             case DOP_SINH_F32: case DOP_TANH_F32: case DOP_ATANH_F32: return 12.0;
                             case DOP_ASINH_F32: case DOP_ACOSH_F32: return 14.0;
                             case DOP_CBRT_F32: return 16.0;
                             case DOP_ERF_F32: case DOP_ERFC_F32: case DOP_ERFINV_F32: return 14.0;
                             case DOP_LGAMMA_F32: case DOP_TGAMMA_F32: return 20.0;
                             case DOP_POW_F32: case DOP_POWR_F32: return 16.0;
                             case DOP_FREXP_M_F32: case DOP_FREXP_E_F32: return 2.0;
                             case DOP_HYPOT_F32: case DOP_HYPOTR_F32: return 8.0;
                             case DOP_DAWSON_F32: return 6.0;
                             case DOP_ERFI_F32: return 14.0;
                             case DOP_CARLSON_RF_F32: case DOP_CARLSON_RD_F32: return 60.0;
                             case DOP_CARLSON_RC_F32: case DOP_CARLSON_RCR_F32: return 40.0;
                             case DOP_SQRT_F32: case DOP_DIV_F32: case DOP_RCP_F32: case DOP_RSQRT_F32: return 3.0; default: return 1.0; } };
        double total_w = 0; for (const EkInstr &in : out.body) total_w += weight(in);
        double acc_w = 0;
        for (size_t i = 0; i + 1 < nb; ++i) {
            acc_w += weight(out.body[i]);
            uint32_t mask = 0; size_t bytes = 0;
            for (size_t k = 0; k < ns; ++k) if (last[k] <= (int) i) { mask |= 1u << k; bytes += out.staged[k].esize; }
            if (!mask) continue;
            double score = ((double) bytes / total_bytes) * ((total_w - acc_w) / total_w);
            if (score > best) { best = score; best_i = (int) i; best_mask = mask; }
        }
        if (best_i >= 0 && best >= 0.15) { out.release_at = best_i; out.release_mask = best_mask; }
    }

    /* rebase uniform indices now that the literal count is known:
       pool = [literals | argument words | scalar pairs] */
    bool finish() {
        uint32_t n_lit = (uint32_t) out.lits.size();
        uint32_t n_arg = (uint32_t) out.argw.size();
        if (n_arg > EK_MAX_ARGW) return fail_resource("too many kernel arguments; call cuda_eval() earlier");
        if (n_lit + n_arg + 2 * out.scalars.size() >= 0x1000u) return fail_resource("uniform pool overflow");
        out.n_tmp = (uint32_t) slot_used.size();
        if (out.n_tmp >= 0x3fffu) return fail_resource("too many live values");
        auto rebase_code = [&](uint16_t code) -> uint16_t {
            if (code == EK_OPND_NONE) return code;
            if (code & 0x8000u) {
                uint32_t i = code & 0x0fffu;
                if (code & 0x2000u) return (uint16_t) (0x8000u | (n_lit + i));
                if (code & 0x1000u) return (uint16_t) (0x8000u | (n_lit + n_arg + i));
                return (uint16_t) (0x8000u | i);
            }
            return code;
        };
        auto fix = [&](std::vector<EkInstr> &v) {
            for (EkInstr &in : v) {
                in.b = rebase_code(in.b); in.c = rebase_code(in.c);
                if (in.flags & EKF_HAS_A) in.a = rebase_code(in.a);
                uint32_t mark = (in.flags >> 12) & 3u;
                in.flags &= ~0x3000u;
                if (mark == 3) {                    /* gather/scatter: low 16 bits = uniform code of pointer */
                    uint16_t code = (uint16_t) (in.imm & 0xffffu);
                    in.imm = (in.imm & 0xffff0000u) | (rebase_code(code) & 0x7fffu);
                } else if (mark == 1) {             /* imm = argument-word index */
                    in.imm = n_lit + (in.imm & 0x0fffu);
                } else if (mark == 2) {             /* dst = argument-word index */
                    in.dst = (uint16_t) (n_lit + (in.dst & 0x0fffu));
                }
            }
        };
        fix(out.init); fix(out.body); fix(out.fini);
        plan_release();
        /* descriptors hold the uniform code of their pointer in word 3: convert to a plain index */
        for (EkInstr &in : out.init) {
            if (in.op == DOP_SMEM_ZERO || in.op == DOP_SMEM_LOAD_TABLE) {
                uint32_t di = in.imm - n_lit;
                uint16_t code = (uint16_t) out.argw[di + 3];
                if (code & 0x8000u) out.argw[di + 3] = rebase_code(code) & 0x7fffu;
            }
        }
        return out.error.empty();
    }
};

/* ------------------------------------------------------------------ planning */
struct Planner {
    EkContext &ctx;
    std::unordered_map<uint32_t, uint32_t> phase_memo;
    std::unordered_set<uint32_t> forced;      /* variables that must be materialised */
    std::map<std::pair<uint32_t, size_t>, Group> groups;   /* (phase, size) */

    explicit Planner(EkContext &c) : ctx(c) {}

    size_t sweep_size(uint32_t idx) const {
        const EkVariable &v = ctx.vars[idx];
        return is_reduce(v.op) ? ctx.vars[v.dep[0]].size : v.size;
    }
    bool is_boundary(uint32_t d, uint32_t consumer) const {
        const EkVariable &dv = ctx.vars[d], &cv = ctx.vars[consumer];
        if (dv.data != nullptr || dv.direct_pointer) return false;
        if (is_reduce(dv.op)) return true;
        size_t csize = is_reduce(cv.op) ? ctx.vars[cv.dep[0]].size : cv.size;
        return dv.size == 1 && csize > 1 && dv.op != EK_OP_LITERAL;
    }

    /* an externally referenced root of an earlier phase is stored by its own launch
       (jit.cu:1165-1169) and can simply be read back instead of being recomputed */
    bool stored_earlier(uint32_t d, uint32_t group_phase) {
        const EkVariable &dv = ctx.vars[d];
        if (dv.data != nullptr || dv.direct_pointer || dv.op == EK_OP_LITERAL) return false;
        if (dv.ref_ext == 0 || dv.side_effect) return false;
        return phase(d) < group_phase;
    }

    uint32_t phase(uint32_t root) {
        /* iterative post-order (tapes can be 10k nodes deep) */
        std::vector<std::pair<uint32_t, int>> stack { { root, 0 } };
        while (!stack.empty()) {
            auto &top = stack.back();
            uint32_t idx = top.first;
            const EkVariable &v = ctx.vars[idx];
            if (phase_memo.count(idx)) { stack.pop_back(); continue; }
            if (v.data != nullptr || v.direct_pointer || v.op == EK_OP_LITERAL) { phase_memo[idx] = 0; stack.pop_back(); continue; }
            if (top.second < 4) {
                uint32_t d = v.dep[top.second++];
                if (d >= EK_REG_RESERVED && !phase_memo.count(d)) stack.push_back({ d, 0 });
                continue;
            }
            uint32_t p = 0;
            for (int k = 0; k < 4; ++k) {
                uint32_t d = v.dep[k];
                if (d < EK_REG_RESERVED) continue;
                p = std::max(p, phase_memo[d] + (is_boundary(d, idx) ? 1u : 0u));
            }
            phase_memo[idx] = p;
            stack.pop_back();
        }
        return phase_memo[root];
    }

    void add_root(uint32_t idx, std::vector<uint32_t> &work) {
        uint32_t p = phase(idx);
        Group &g = groups[{ p, sweep_size(idx) }];
        g.phase = p; g.size = sweep_size(idx);
        collect(g, idx, &work);
    }

    /* DFS post-order from `idx` into group `g`, heavier subtree first (jit.cu:1385-1416) */
    void collect(Group &g, uint32_t idx, std::vector<uint32_t> *work) {
        if (g.visited.count(idx)) return;
        struct Frame { uint32_t idx; uint32_t deps[4]; int n; int i; };
        std::vector<Frame> stack;
        auto push = [&](uint32_t i) {
            if (g.visited.count(i)) return;
            g.visited.insert(i);
            Frame f; f.idx = i; f.n = 0; f.i = 0;
            const EkVariable &v = ctx.vars[i];
            if (v.data == nullptr && !v.direct_pointer) {
                for (int k = 0; k < 4; ++k) if (v.dep[k] >= EK_REG_RESERVED) f.deps[f.n++] = v.dep[k];
                std::stable_sort(f.deps, f.deps + f.n, [&](uint32_t a, uint32_t b) {
                    return ctx.vars[a].subtree_size > ctx.vars[b].subtree_size; });
            }
            stack.push_back(f);
        };
        push(idx);
        while (!stack.empty()) {
            Frame &f = stack.back();
            if (f.i < f.n) {
                uint32_t d = f.deps[f.i++];
                if (is_boundary(d, f.idx) || stored_earlier(d, g.phase)) {
                    /* produced by an earlier launch: becomes an input here and a root there */
                    if (!forced.count(d)) { forced.insert(d); if (work) work->push_back(d); }
                    if (!g.visited.count(d)) {
                        g.sched.push_back(d);          /* appears in the schedule as an input */
                        g.visited.insert(d);
                        g.boundary.insert(d);
                    }
                } else push(d);
                continue;
            }
            g.sched.push_back(f.idx);
            stack.pop_back();
        }
        g.roots.push_back(idx);
    }
};

/* Layout of the 'extra' shared-memory region for one configuration.  General kernels: the assembly-time layout.
   Fast kernel (V = 16): scatter_add bins of up to 32 KB get ONE PRIVATE COPY PER THREAD (integer as well as float bins:
   plain LDS / add / STS, bank = thread id whatever the bin -- no shared-memory atomics); larger targets keep the
   [bin][copy] layout with up to 32 copies updated atomically.  Returns the size; writes offsets / copy counts into
   `argw` when it is given. */
uint32_t fast_copies(uint32_t count, uint32_t T) {
    return (uint64_t) count * T * 4u <= 32768u ? T : std::max(1u, std::min(32u, 4096u / count));
}
size_t layout_extra(const Assembled &a, const Config &cfg, uint32_t *argw) {
    if (!cfg.fast) return a.extra_bytes;
    uint32_t off = 0;
    for (const Assembled::ExtraItem &it : a.extra_items) {
        uint32_t copies = it.kind == 0 ? 1u : fast_copies(it.count, cfg.T);
        if (argw) { argw[it.di] = off; argw[it.di + 2] = copies; }
        off += (it.count * copies * 4u + 15u) & ~15u;
    }
    return off;
}

size_t smem_layout(const Assembled &a, Config &cfg, size_t n_uni) {
    size_t off = n_uni * 16;                        /* every uniform word is replicated 4x */
    cfg.off_bar = (uint32_t) off; off += 8 * 8 + 33 * 8;
    off = (off + 15) & ~(size_t) 15;
    size_t n_prog = a.init.size() + a.body.size() + a.fini.size();
    cfg.prog_in_smem = !cfg.fast && n_prog * 16 <= 24 * 1024;
    cfg.off_prog = (uint32_t) off;
    if (cfg.prog_in_smem) off += n_prog * 16;
    cfg.off_extra = (uint32_t) off; off += layout_extra(a, cfg, nullptr);
    off = (off + 1023) & ~(size_t) 1023;
    cfg.off_slots = (uint32_t) off;
    size_t slot_bytes = (size_t) cfg.T * cfg.V * 4;
    off += slot_bytes * (a.n_tmp + (size_t) cfg.stages * a.n_in_units);
    cfg.smem = off;
    return off;
}

/* ---- lowering for the 32-bit fast kernel (ek_sweep_fast.cu; format: ek_isa.h "lowered instruction format") ---- */
int fop_of(int dop) {
    switch (dop) {
        case DOP_NOP: return FOP_NOP;
#define X(n) case DOP_##n: return FOP_##n;
        EK_FOPS2(X)
        X(FMA_F32) X(FMAC_F32) X(MAD_I32) X(MADC_I32) X(FMANZ_F32) X(FMANZC_F32) X(SEL_M_32) X(SEL_T_32) X(SEL_F_32)
        X(ABS_F32) X(NEG_F32) X(SQRT_F32) X(RCP_F32) X(RSQRT_F32) X(EXP_F32) X(LOG_F32) X(SIN_F32) X(COS_F32)
        X(FLOOR_F32) X(CEIL_F32) X(ROUND_F32) X(TRUNC_F32) X(ABS_I32) X(NEG_I32) X(NOT_32) X(NOT_B) X(NEZ_32)
        X(CVT_F32_I32) X(CVT_F32_U32) X(CVT_I32_F32) X(CVT_U32_F32)
        X(INDEX) X(LD_U8) X(LD_S8) X(LDG_32) X(ST_32) X(ST_8)
        X(GATHER_32) X(GATHER_32_SMEM) X(SCATTER_32) X(SCATTER_ADD_F32) X(SCATTER_ADD_I32)
        X(SCATTER_ADD_F32_SMEM) X(SCATTER_ADD_I32_SMEM) X(RACC)
        EK_FOPS0(X)
        X(TAN_F32) X(COT_F32) X(ASIN_F32) X(ACOS_F32) X(ATAN_F32) X(ATAN2_F32) X(ATAN2R_F32)
        X(SINH_F32) X(COSH_F32) X(TANH_F32) X(ASINH_F32) X(ACOSH_F32) X(ATANH_F32) X(CBRT_F32)
        X(ERF_F32) X(ERFC_F32) X(ERFINV_F32) X(LGAMMA_F32) X(TGAMMA_F32)
        X(POW_F32) X(POWR_F32) X(FREXP_M_F32) X(FREXP_E_F32) X(HYPOT_F32) X(HYPOTR_F32) X(DAWSON_F32) X(ERFI_F32)
        X(CARLSON_RF_F32) X(CARLSON_RD_F32) X(CARLSON_RC_F32) X(CARLSON_RCR_F32)
#undef X
        case DOP_LOAD_32: return FOP_LOAD;
        default: return -1;
    }
}
bool fop_has_u_twin(int fop) {
    switch (fop) {
#define X(n) case FOP_##n:
        EK_FOPS2(X)
#undef X
        case FOP_ATAN2_F32: case FOP_ATAN2R_F32:
        case FOP_POW_F32: case FOP_POWR_F32: case FOP_HYPOT_F32: case FOP_HYPOTR_F32:
            return true;
        default: return false;
    }
}

/* `in` = assembled instructions whose operand codes are still symbolic (uniform index | 0x8000, staged unit | 0x4000,
   temporary slot); cfg == nullptr: count / check only.  Appends to `out`; false = not expressible.  release_at >= 0
   (the body, with a.release_at): a NOP carrying FF_REL and the release mask (imm) follows what in[release_at] lowers to. */
bool lower_fast(const std::vector<EkInstr> &in, const Assembled &a, const Config *cfg, std::vector<EkInstr> &out, int release_at = -1) {
    const uint32_t slot_bytes = cfg ? cfg->T * 16u * 4u : 0u;
    auto is_uni = [](uint16_t c) { return c != EK_OPND_NONE && (c & EK_OPND_UNI) != 0; };
    /* per-thread operand -> absolute byte offset >> 4; uniform operand -> pool word index */
    auto enc = [&](uint16_t c) -> uint16_t {
        if (c == EK_OPND_NONE) return 0;
        if (c & EK_OPND_UNI) return (uint16_t) (c & 0x7fffu);
        if (!cfg) return 0;
        uint32_t off = (c & EK_OPND_STAGED) ? cfg->off_slots + (a.n_tmp + (c & 0x3fffu)) * slot_bytes
                                            : cfg->off_slots + (uint32_t) c * slot_bytes;
        return (uint16_t) (off >> 4);
    };
    auto emit = [&](uint32_t fop, uint32_t fl, uint16_t b, uint16_t c, uint16_t dst, uint16_t aux, uint32_t imm) {
        EkInstr o;
        o.op = (uint16_t) fop; o.flags = (uint16_t) fl; o.dst = b; o.b = c; o.c = dst; o.a = aux; o.imm = imm;
        /* (EkInstr field order = word layout x = op | flags << 16, y = dst | b << 16, z = c | a << 16: the lowered
           format reads y = b | c << 16, z = dst | aux << 16 -- hence the shuffled assignment above) */
        out.push_back(o);
    };
    const size_t first = out.size();
    /* (emitted once every instruction lowered from in[release_at] is out: at the top of the next iteration) */
    bool released = false;
    auto mark_release = [&](size_t j) {
        if (!released && release_at >= 0 && j > (size_t) release_at) { emit(FOP_NOP, FF_REL, 0, 0, 0, 0, a.release_mask); released = true; }
    };
    for (size_t j = 0; j < in.size(); ++j) {
        mark_release(j);
        const EkInstr &i = in[j];
        if (i.flags & (EKF_R64 | EKF_B64 | EKF_C64 | EKF_A64)) return false;
        /* 1. accumulator load and input modifiers become instructions of their own */
        if (i.flags & EKF_HAS_A) {
            if (is_uni(i.a)) emit(FOP_LOADU, 0, enc(i.a), 0, 0, 0, 0);
            else emit(FOP_LOAD, 0, enc(i.a), 0, 0, 0, 0);
        }
        /* (|x| is applied before -x, like the general kernel does; exp(-x) and sqrt(|x|) have fused forms) */
        const bool fuse_neg = i.op == DOP_EXP_F32 && (i.flags & EKF_NEG_A) && !(i.flags & EKF_ABS_A);
        const bool fuse_abs = i.op == DOP_SQRT_F32 && (i.flags & EKF_ABS_A) && !(i.flags & EKF_NEG_A);
        if ((i.flags & EKF_ABS_A) && !fuse_abs) emit(FOP_ABS_F32, 0, 0, 0, 0, 0, 0);
        if ((i.flags & EKF_NEG_A) && !fuse_neg) emit(FOP_NEG_F32, 0, 0, 0, 0, 0, 0);
        /* 2. the operation */
        int fop = fuse_neg ? FOP_EXPN_F32 : fuse_abs ? FOP_SQRTA_F32 : fop_of(i.op);
        /* Float16 storage: a staged input read by its conversion (LD_U16; CVT_F16_F32) and an output stored by its
           conversion (CVT_F32_F16; ST_16, when the next instruction reloads the accumulator or there is none: FOP_ST_F16
           leaves the accumulator as it was) are one operation each; any other 16-bit instruction has no fast form.
           `post` is the instruction whose post actions and imm the lowered operation carries. */
        const EkInstr *post = &i;
        if (j + 1 < in.size()) {
            const EkInstr &nx = in[j + 1];
            if (i.op == DOP_LD_U16 && i.flags == 0 && nx.op == DOP_CVT_F16_F32 &&
                !(nx.flags & (EKF_HAS_A | EKF_NEG_A | EKF_ABS_A | EKF_HAS_B | EKF_HAS_C))) { fop = FOP_LD_F16; post = &nx; ++j; }
            else if (i.op == DOP_CVT_F32_F16 && !(i.flags & (EKF_ST | EKF_STG | EKF_RACC)) && nx.op == DOP_ST_16 && nx.flags == 0 &&
                     (j + 2 == in.size() || (in[j + 2].flags & EKF_HAS_A))) {
                fop = FOP_ST_F16; post = &nx; ++j;
            }
        }
        if (fop < 0) return false;
        uint32_t fl = 0;
        uint16_t b = 0, c = 0, dst = 0, aux = 0;
        const bool hb = (i.flags & EKF_HAS_B) != 0, hc = (i.flags & EKF_HAS_C) != 0;
        const bool ub = hb && is_uni(i.b), uc = hc && is_uni(i.c);
        if (hb) b = enc(i.b);
        if (hc) c = enc(i.c);
        switch (i.op) {
            case DOP_LOAD_32:                                     /* R = B */
                if (!hb) return false;
                fop = ub ? FOP_LOADU : FOP_LOAD;
                break;
            case DOP_LD_U8: case DOP_LD_S8: case DOP_LD_U16:      /* raw staged code in b, no EKF_HAS_B (LD_U16: FOP_LD_F16) */
                b = enc(i.b);
                break;
            case DOP_GATHER_32: case DOP_GATHER_32_SMEM:          /* mask = B */
                if (!hb) return false;
                fl |= ub ? FF_MU : FF_B;
                break;
            case DOP_SCATTER_32: case DOP_SCATTER_ADD_F32: case DOP_SCATTER_ADD_I32:
            case DOP_SCATTER_ADD_F32_SMEM: case DOP_SCATTER_ADD_I32_SMEM:     /* value = B, mask = C */
                if (!hb || !hc) return false;
                fl |= ub ? FF_VU : FF_B;
                fl |= uc ? FF_MU : FF_C;
                break;
            case DOP_FMA_F32:
                if (ub && !uc) { fop = FOP_FMA_F32_UB; fl |= FF_C; }
                else if (uc && !ub) { fop = FOP_FMA_F32_UC; fl |= FF_B; }
                else if (ub && uc) { fop = FOP_FMA_F32_UB; fl |= FF_CU; }
                else fl |= FF_B | FF_C;
                break;
            case DOP_FMAC_F32:                                    /* B * C + R (commutative in B, C) */
                if (ub && !uc) { fop = FOP_FMAC_F32_UB; fl |= FF_C; }
                else if (uc && !ub) { fop = FOP_FMAC_F32_UB; std::swap(b, c); fl |= FF_C; }
                else if (ub && uc) { fop = FOP_FMAC_F32_UB; fl |= FF_CU; }
                else fl |= FF_B | FF_C;
                break;
            case DOP_RFIN:                                        /* b = slot of the partials, dst = pool index of the pointer */
                if (!hb || ub) return false;
                dst = i.dst;
                break;
            case DOP_SMEM_ZERO:                                   /* dst = 1: float bins (filled with -0.0) */
                dst = i.dst;
                break;
            default:
                if (hb && ub && !hc && fop_has_u_twin(fop)) fop += 1;          /* X_U (X_UB) = X + 1 */
                else {
                    if (hb) fl |= ub ? FF_BU : FF_B;
                    if (hc) fl |= uc ? FF_CU : FF_C;
                }
                break;
        }
        /* 3. post actions */
        const EkInstr &p = *post;
        if (p.flags & EKF_ST) { fl |= FF_ST; dst = enc(p.dst); }
        if (p.flags & EKF_STG) fl |= FF_STG;
        if ((p.flags & EKF_RACC) || p.op == DOP_RACC) {
            if (p.flags & EKF_ST) return false;
            fl |= FF_RACC; dst = enc(p.dst);
            aux = (uint16_t) (p.op == DOP_RACC ? (p.imm & 0xffffu) : p.a);
            if (((aux >> 8) & 0xffu) > EK_RC_U32) return false;
        }
        if (i.op == DOP_NOP && !fl) continue;                    /* (a bare carrier of a load / modifier) */
        emit((uint32_t) fop, fl, b, c, dst, aux, p.imm);
    }
    mark_release(in.size());
    return true;
}

/* a program as one kernel reads it */
struct Program {
    std::vector<EkInstr> init, body, fini;
    size_t size() const { return init.size() + body.size() + fini.size(); }
};

/* lower_fast on all three sections (the body with its release NOP) */
bool lower_fast_all(const Assembled &a, const Config *cfg, Program &p) {
    return lower_fast(a.init, a, cfg, p.init) && lower_fast(a.body, a, cfg, p.body, a.release_at) && lower_fast(a.fini, a, cfg, p.fini);
}

/* the program the kernel of `cfg` receives: for the general kernels the operand codes become (byte offset >> 4) in
   this configuration's shared-memory layout; for the fast kernel, the lowered form */
bool kernel_program(const Assembled &a, const Config &cfg, Program &p) {
    if (cfg.fast) return lower_fast_all(a, &cfg, p);
    const uint32_t slot_bytes = cfg.T * cfg.V * 4u;
    auto patch = [&](uint16_t code) -> uint16_t {
        if (code == EK_OPND_NONE || (code & EK_OPND_UNI)) return code;      /* uniform index == offset >> 4 */
        if (code & EK_OPND_STAGED) return (uint16_t) (EK_OPND_STAGED | (((code & 0x3fffu) * slot_bytes) >> 4));
        return (uint16_t) ((cfg.off_slots + (uint32_t) code * slot_bytes) >> 4);
    };
    auto patch_all = [&](const std::vector<EkInstr> &from, std::vector<EkInstr> &v) {
        v = from;
        for (EkInstr &in : v) {
            in.b = patch(in.b); in.c = patch(in.c);
            if (in.flags & EKF_HAS_A) in.a = patch(in.a);
            if ((in.flags & (EKF_ST | EKF_RACC)) || in.op == DOP_RACC) in.dst = patch(in.dst);
        }
    };
    patch_all(a.init, p.init); patch_all(a.body, p.body); patch_all(a.fini, p.fini);
    return true;
}

/* the argument words the kernel of `cfg` receives, pointer words not yet filled in */
void argument_words(const Assembled &a, const Config &cfg, uint32_t *argw) {
    if (!a.argw.empty()) memcpy(argw, a.argw.data(), a.argw.size() * 4);
    layout_extra(a, cfg, argw);
}

/* kernel configurations, tried in order (V, T, stages, CTAs per SM) */
struct Cand { int V; uint32_t T; uint32_t stages; uint32_t want_ctas; };
/* the 32-bit fast kernel: V = 16, one TMA stage (the other CTAs of the SM hide the load) */
const Cand fast_cands[] = { { 16, 256, 1, 2 }, { 16, 128, 1, 4 }, { 16, 128, 1, 3 }, { 16, 128, 1, 2 }, { 16, 256, 1, 1 }, { 16, 128, 1, 1 } };
const Cand wide_cands[] = {
    /* the general kernel: single-buffered staging with more resident CTAs first, double buffering after: the
       other CTAs of the SM hide the TMA latency and 16 warps hide the interpreter's dependent-issue latency */
    { 8, 256, 1, 4 }, { 8, 256, 1, 3 }, { 8, 256, 2, 2 }, { 8, 256, 1, 2 }, { 8, 256, 2, 1 }, { 8, 256, 1, 1 },
    /* (no { 8, 128, 1, 2 }: a program that { 8, 256, 1, 1 } rejects needs more than half of an SM's shared memory at
       T = 128, so two such CTAs never fit) */
    { 8, 128, 2, 1 }, { 8, 128, 1, 1 },
    { 4, 128, 2, 1 }, { 4, 64, 2, 1 }, { 4, 32, 2, 1 } };
/* tiny sweeps (incl. the size-1 scalar groups): one small CTA */
const Cand small_cands[] = { { 4, 32, 2, 1 }, { 4, 128, 2, 1 }, { 8, 256, 2, 1 } };

bool choose_config(const EkContext &ctx, const Assembled &a, size_t n, Config &cfg, std::string &err) {
    size_t n_uni = a.lits.size() + a.argw.size() + 2 * a.scalars.size();
    size_t budget = ctx.smem_optin;                 /* per CTA (227 KB) */
    size_t per_sm = 228 * 1024 - 1024;              /* per SM, minus the 1 KB per-CTA reservation */
    const bool fast_ok = ctx.fast_mode != 0 && !a.has64 && a.fast_ok && a.fast_len <= EK_INLINE_PROG;
    cfg.fast = false;
    if (n <= 4096) {
        uint32_t pick = n <= 128 ? 0 : n <= 512 ? 1 : 2;
        for (uint32_t k = pick; k < 3; ++k) {
            cfg.V = small_cands[k].V; cfg.T = small_cands[k].T; cfg.stages = 2; cfg.ctas_per_sm = 1;
            if (smem_layout(a, cfg, n_uni) <= budget) return true;
        }
    }
    if (fast_ok) {
        /* testing aid: EK_FAST_T=128 / 256 restricts the fast kernel to one block size (tests/test_cpu_fast_kernel.py runs
           the host-compiled kernel on both instantiations) */
        static const int only_T = getenv("EK_FAST_T") ? atoi(getenv("EK_FAST_T")) : 0;
        for (const Cand &c : fast_cands) {
            if (only_T && (int) c.T != only_T) continue;
            cfg.fast = true;
            cfg.V = c.V; cfg.T = c.T; cfg.stages = 1; cfg.ctas_per_sm = c.want_ctas;
            size_t need = smem_layout(a, cfg, n_uni);
            if (need > budget) continue;
            if ((need + 1024) * c.want_ctas > per_sm + 1024) continue;
            return true;
        }
        cfg.fast = false;
    }
    for (const Cand &c : wide_cands) {
        cfg.V = c.V; cfg.T = c.T; cfg.stages = a.n_in_units ? c.stages : 2; cfg.ctas_per_sm = c.want_ctas;
        size_t need = smem_layout(a, cfg, n_uni);
        if (need > budget) continue;
        if ((need + 1024) * c.want_ctas > per_sm + 1024) continue;
        return true;
    }
    err = "expression too large for one kernel (" + std::to_string(a.n_tmp) + " live values, " +
          std::to_string(a.n_in_units) + " input streams); insert cuda_eval() to split it";
    return false;
}

uint64_t fnv1a(const uint8_t *p, size_t n) {
    uint64_t h = 1469598103934665603ull;
    for (size_t i = 0; i < n; ++i) { h ^= p[i]; h *= 1099511628211ull; }
    return h;
}

/* device copies of programs / literal pools that do not fit the kernel parameters (rare: > 448 instructions or > 128
   literal words).  Keyed on exactly what is uploaded; bounded: the cache is emptied when it reaches 256 entries (the
   stream is synchronised first, so no launch still reads the freed buffers). */
void lookup_program(EkContext &ctx, const Program &prog, const std::vector<uint32_t> &lits, bool need_prog, bool need_lit,
                    const EkInstr *&d_prog, const uint32_t *&d_lit) {
    std::vector<uint8_t> key;
    auto append = [&](const void *p, size_t n) { const uint8_t *b = (const uint8_t *) p; key.insert(key.end(), b, b + n); };
    uint32_t hdr[4] = { need_prog ? (uint32_t) prog.init.size() : 0u, need_prog ? (uint32_t) prog.body.size() : 0u,
                        need_prog ? (uint32_t) prog.fini.size() : 0u, need_lit ? (uint32_t) lits.size() : 0u };
    append(hdr, sizeof(hdr));
    if (need_prog) {
        append(prog.init.data(), prog.init.size() * sizeof(EkInstr));
        append(prog.body.data(), prog.body.size() * sizeof(EkInstr));
        append(prog.fini.data(), prog.fini.size() * sizeof(EkInstr));
    }
    if (need_lit) append(lits.data(), lits.size() * 4);
    uint64_t h = fnv1a(key.data(), key.size());
    {
        auto it = ctx.programs.find(h);
        if (it != ctx.programs.end())
            for (auto &e : it->second) if (e.key == key) { d_prog = e.d_prog; d_lit = e.d_lit; return; }
    }
    size_t entries = 0;
    for (auto &kv : ctx.programs) entries += kv.second.size();
    if (entries >= 256) {
        ek_cuda_check(cudaStreamSynchronize(ctx.stream));
        for (auto &kv : ctx.programs) for (auto &e : kv.second) { if (e.d_prog) cudaFree(e.d_prog); if (e.d_lit) cudaFree(e.d_lit); }
        ctx.programs.clear();
    }
    EkProgramCacheEntry e;
    e.key = key;
    e.d_prog = nullptr; e.d_lit = nullptr;
    if (need_prog) {
        std::vector<EkInstr> all;
        all.insert(all.end(), prog.init.begin(), prog.init.end());
        all.insert(all.end(), prog.body.begin(), prog.body.end());
        all.insert(all.end(), prog.fini.begin(), prog.fini.end());
        ek_cuda_check(cudaMalloc(&e.d_prog, std::max<size_t>(all.size(), 1) * sizeof(EkInstr)));
        /* synchronous copies from pageable memory: only on a cache miss */
        if (!all.empty()) ek_cuda_check(cudaMemcpy(e.d_prog, all.data(), all.size() * sizeof(EkInstr), cudaMemcpyHostToDevice));
    }
    if (need_lit) {
        ek_cuda_check(cudaMalloc(&e.d_lit, std::max<size_t>(lits.size(), 1) * 4));
        if (!lits.empty()) ek_cuda_check(cudaMemcpy(e.d_lit, lits.data(), lits.size() * 4, cudaMemcpyHostToDevice));
    }
    d_prog = e.d_prog; d_lit = e.d_lit;
    ctx.programs[h].push_back(std::move(e));
}

const char *dop_name(uint16_t op) {
    static const char *names[] = {
#define X(n) #n,
        EK_DOPS(X)
#undef X
    };
    return op < DOP__COUNT ? names[op] : "?";
}

std::string opnd_str(uint16_t c) {
    if (c == EK_OPND_NONE) return "-";
    if (c & 0x8000u) return "u" + std::to_string(c & 0x3fffu);
    if (c & EK_OPND_STAGED) return "in" + std::to_string(c & 0x3fffu);
    return "s" + std::to_string(c);
}

void dump_program(std::ostream &os, const Assembled &a, const Group &g) {
    os << "sweep phase=" << g.phase << " n=" << g.size << " in=" << a.staged.size() << " scalars=" << a.scalars.size()
       << " out=" << a.outputs.size() << " ops=" << a.n_arith << " tmp_slots=" << a.n_tmp << " lits=" << a.lits.size() << "\n";
    auto sec = [&](const char *name, const std::vector<EkInstr> &v) {
        for (const EkInstr &in : v) {
            os << "  " << name << " " << dop_name(in.op);
            if (in.flags & EKF_HAS_A) os << " a=" << opnd_str(in.a);
            if (in.flags & EKF_NEG_A) os << " neg";
            if (in.flags & EKF_ABS_A) os << " abs";
            os << " b=" << opnd_str(in.b) << " c=" << opnd_str(in.c);
            if (in.flags & EKF_STG) os << " stg";
            if (in.flags & EKF_RACC) os << " racc->s" << in.dst;
            if (in.flags & EKF_ST) os << " -> s" << in.dst;
            os << " imm=0x" << std::hex << in.imm << std::dec << "\n";
        }
    };
    sec("init", a.init); sec("body", a.body); sec("fini", a.fini);
}

/* ------------------------------------------------------------------ the sweeps of one eval */
/* one kernel launch: a group, its assembled program (operand codes still symbolic) and the configuration it runs with */
struct Sweep { Group *g; Assembled a; Config cfg; };

/* what ek_eval() launches for the live set, in launch order, together with the groups the sweeps point into */
struct Schedule {
    Planner plan;
    std::vector<std::unique_ptr<Group>> split_groups;
    std::vector<Sweep> sweeps;
    std::vector<uint32_t> kept_literals;      /* live literals: no sweep computes them, they stay live */
    std::vector<uint32_t> prints;             /* print nodes (EK_OP_PRINTF), in recording order */

    explicit Schedule(EkContext &ctx) : plan(ctx) {}

    /* assemble every group before anything is launched, so that user errors leave the trace untouched */
    bool build() {
        EkContext &ctx = plan.ctx;
        /* Roots are planned in CREATION order: the reference walks a std::set of monotonically increasing ids
           (jit.cu:1385-1416), so of two scatters into the same target the one recorded later runs later and wins, a
           scatter recorded after a gather from the same array comes after it, and so on.  Handles are recycled here, so
           the order is the per-variable sequence number, not the handle. */
        std::vector<uint32_t> work(ctx.live.begin(), ctx.live.end());
        std::sort(work.begin(), work.end(), [&](uint32_t a, uint32_t b) { return ctx.vars[a].seq > ctx.vars[b].seq; });
        while (!work.empty()) {                              /* (pop_back: oldest first) */
            uint32_t idx = work.back(); work.pop_back();
            const EkVariable &v = ctx.vars[idx];
            if (!v.used) continue;
            if (v.data != nullptr && !v.side_effect) continue;
            /* a print computes nothing itself: each computed argument becomes a root that its sweep must store (the
               existing output store materialises it); evaluated and literal arguments are read as they are */
            if (v.op == EK_OP_PRINTF) {
                prints.push_back(idx);
                for (int k = 0; k < 3; ++k) {
                    uint32_t d = v.dep[k];
                    if (d < EK_REG_RESERVED) continue;
                    const EkVariable &dv = ctx.vars[d];
                    if (dv.data != nullptr || dv.direct_pointer || dv.op == EK_OP_LITERAL) continue;
                    plan.forced.insert(d);
                    plan.add_root(d, work);
                }
                continue;
            }
            /* literals are immediates: they are only given storage on demand (ek_eval_var) */
            if (v.op == EK_OP_LITERAL) { kept_literals.push_back(idx); continue; }
            plan.add_root(idx, work);
        }
        for (auto &kv : plan.groups)                         /* ordered by (phase asc, size asc) */
            if (!assemble(kv.second)) return false;
        /* within a phase launch the largest size first (jit.cu:1450) */
        std::stable_sort(sweeps.begin(), sweeps.end(), [](const Sweep &a, const Sweep &b) {
            if (a.g->phase != b.g->phase) return a.g->phase < b.g->phase;
            return a.g->size > b.g->size; });
        return true;
    }

    /* assemble `g`; when a per-kernel limit is hit (slots, inputs, arguments ...) split its roots in
       two and retry -- shared sub-expressions are then recomputed, exactly as the reference does
       across kernels of different sizes */
    bool assemble(Group &g) {
        if (g.sched.empty()) return true;
        if (g.size > 0xffffffffull) { ek_set_error("ek_eval(): arrays with more than 2^32-1 entries are not supported (jit.cu:1066,1090)"); return false; }
        Assembler as(plan.ctx, g, plan.forced);
        bool ok = as.run();
        if (ok && !as.out.has64) {
            Program lowered;
            as.out.fast_ok = lower_fast_all(as.out, nullptr, lowered);
            as.out.fast_len = (uint32_t) lowered.size();
        }
        Config cfg; std::string cerr;
        if (ok && !choose_config(plan.ctx, as.out, g.size, cfg, cerr)) { ok = false; as.out.error = cerr; as.out.resource_error = true; }
        if (ok) { sweeps.push_back({ &g, std::move(as.out), cfg }); return true; }
        if (!as.out.resource_error || g.roots.size() < 2) { ek_set_error("ek_eval(): " + as.out.error); return false; }
        size_t half = g.roots.size() / 2;
        for (int part = 0; part < 2; ++part) {
            split_groups.emplace_back(new Group());
            Group &sub = *split_groups.back();
            sub.phase = g.phase; sub.size = g.size;
            size_t lo = part == 0 ? 0 : half, hi = part == 0 ? half : g.roots.size();
            for (size_t r = lo; r < hi; ++r) plan.collect(sub, g.roots[r], nullptr);
            if (!assemble(sub)) return false;
        }
        return true;
    }
};

/* `s` as a JSON string literal (the print formats of the dry runs) */
void json_string(std::ostream &os, const std::string &s) {
    os << '"';
    for (unsigned char c : s) {
        if (c == '"' || c == '\\') os << '\\' << c;
        else if (c == '\n') os << "\\n";
        else if (c == '\t') os << "\\t";
        else if (c < 0x20) { char b[8]; snprintf(b, sizeof(b), "\\u%04x", c); os << b; }
        else os << c;
    }
    os << '"';
}

/* machine-readable form of the ek_debug_plan() listing for tests/ek_emulator.py (a numpy interpreter of the sweep ISA
   that lets the CPU test-suite execute what the planner + assembler produce) */
void write_program_json(std::ostream &os, const EkContext &ctx, const std::vector<Sweep> &sweeps, const std::vector<uint32_t> &prints) {
    auto instrs = [&](const char *name, const std::vector<EkInstr> &v) {
        os << ",\"" << name << "\":[";
        for (size_t i = 0; i < v.size(); ++i)
            os << (i ? "," : "") << "[" << v[i].op << "," << v[i].flags << "," << v[i].dst << "," << v[i].b << "," << v[i].c << "," << v[i].a << "," << v[i].imm << "]";
        os << "]";
    };
    os << "{\"ops\":[";
    for (int k = 0; k < DOP__COUNT; ++k) os << (k ? "," : "") << "\"" << dop_name((uint16_t) k) << "\"";
    os << "],\"sweeps\":[";
    for (size_t si = 0; si < sweeps.size(); ++si) {
        const Sweep &s = sweeps[si];
        const Assembled &a = s.a;
        os << (si ? "," : "") << "{\"phase\":" << s.g->phase << ",\"n\":" << s.g->size << ",\"n_tmp\":" << a.n_tmp;
        instrs("init", a.init); instrs("body", a.body); instrs("fini", a.fini);
        os << ",\"lits\":[";
        for (size_t i = 0; i < a.lits.size(); ++i) os << (i ? "," : "") << a.lits[i];
        os << "],\"argw\":[";
        for (size_t i = 0; i < a.argw.size(); ++i) os << (i ? "," : "") << a.argw[i];
        os << "],\"ptr_fix\":[";
        for (size_t i = 0; i < a.ptr_fix.size(); ++i) os << (i ? "," : "") << "[" << a.ptr_fix[i].argw << "," << a.ptr_fix[i].var << "," << (a.ptr_fix[i].output ? 1 : 0) << "," << (unsigned long long) (uintptr_t) ctx.vars[a.ptr_fix[i].var].data << "]";
        os << "],\"staged\":[";
        for (size_t i = 0; i < a.staged.size(); ++i) os << (i ? "," : "") << "[" << a.staged[i].var << "," << a.staged[i].unit << "," << (int) a.staged[i].esize << "]";
        os << "],\"scalars\":[";
        for (size_t i = 0; i < a.scalars.size(); ++i) os << (i ? "," : "") << "[" << a.scalars[i].var << "," << (int) ctx.vars[a.scalars[i].var].type << "]";
        os << "],\"outputs\":[";
        for (size_t i = 0; i < a.outputs.size(); ++i) os << (i ? "," : "") << "[" << a.outputs[i].var << "," << a.outputs[i].argw << "," << a.outputs[i].bytes << "," << (int) ctx.vars[a.outputs[i].var].type << "]";
        os << "]";
        /* the configuration this sweep launches with, and the program it sends */
        Program prog;
        const bool expressible = kernel_program(a, s.cfg, prog);
        os << ",\"config\":{\"fast\":" << (s.cfg.fast ? 1 : 0) << ",\"V\":" << s.cfg.V << ",\"T\":" << s.cfg.T
           << ",\"stages\":" << s.cfg.stages << ",\"ctas_per_sm\":" << s.cfg.ctas_per_sm << ",\"smem\":" << s.cfg.smem
           << ",\"prog_in_smem\":" << (s.cfg.prog_in_smem ? 1 : 0)
           << ",\"inline_prog\":" << (prog.size() <= EK_INLINE_PROG ? 1 : 0)
           << ",\"inline_lit\":" << (a.lits.size() <= EK_MAX_LIT_INLINE ? 1 : 0) << "}";
        /* the program as the 32-bit fast kernel receives it: this sweep's own when it runs there; otherwise the one it
           would receive if the sweep were wide (so that small CPU test cases exercise the lowering too), when the
           launcher would then pick the fast kernel */
        Config fcfg = s.cfg; Program fprog; std::string ferr;
        const Program *fast = s.cfg.fast && expressible ? &prog : nullptr;
        if (!s.cfg.fast && choose_config(ctx, a, std::max<size_t>(s.g->size, 4097), fcfg, ferr) && fcfg.fast && kernel_program(a, fcfg, fprog))
            fast = &fprog;
        if (fast) {
            os << ",\"fast\":{\"T\":" << fcfg.T << ",\"off_slots\":" << fcfg.off_slots << ",\"n_tmp\":" << a.n_tmp
               << ",\"off_bar\":" << fcfg.off_bar << ",\"off_extra\":" << fcfg.off_extra << ",\"smem\":" << fcfg.smem
               << ",\"n_in_units\":" << a.n_in_units << ",\"n_red\":" << a.n_red << ",\"argw\":[";
            std::vector<uint32_t> aw(a.argw.size());
            argument_words(a, fcfg, aw.data());
            for (size_t i = 0; i < aw.size(); ++i) os << (i ? "," : "") << aw[i];
            os << "]";
            /* (fop, fflags, b, c, dst, aux, imm): see the field shuffle in lower_fast */
            instrs("init", fast->init); instrs("body", fast->body); instrs("fini", fast->fini);
            /* ext: the EK_FX_* operation sets of the body, i.e. the instantiation ek_fast_kernel<T, ext> that runs it */
            os << ",\"release_mask\":" << (a.release_at >= 0 ? a.release_mask : 0u)
               << ",\"ext\":" << ek_fast_ext(fast->body.data(), (uint32_t) fast->body.size()) << "}";
        }
        os << "}";
    }
    os << "],\"configs\":{";
    {   /* the candidate lists of choose_config, in the order it tries them */
        auto cl = [&](const char *name, const Cand *c, size_t k, bool last) {
            os << "\"" << name << "\":[";
            for (size_t i = 0; i < k; ++i) os << (i ? "," : "") << "[" << c[i].V << "," << c[i].T << "," << c[i].stages << "," << c[i].want_ctas << "]";
            os << "]" << (last ? "" : ",");
        };
        cl("small", small_cands, sizeof(small_cands) / sizeof(Cand), false);
        cl("fast", fast_cands, sizeof(fast_cands) / sizeof(Cand), false);
        cl("wide", wide_cands, sizeof(wide_cands) / sizeof(Cand), true);
    }
    os << "},\"fops\":[";
    {
        static const char *fnames[] = { "NOP",
#define X(n) #n, #n "_U",
            EK_FOPS2(X)
#undef X
#define X(n) #n,
            EK_FOPS1(X) EK_FOPS0(X) EK_FOPS16(X) EK_FOPST(X) EK_FOPSH(X) EK_FOPSS(X) EK_FOPSM(X) EK_FOPSE(X)
#undef X
        };
        for (int k = 0; k < FOP__COUNT; ++k) os << (k ? "," : "") << "\"" << fnames[k] << "\"";
    }
    os << "],\"prints\":[";
    for (size_t i = 0; i < prints.size(); ++i) {
        const EkVariable &v = ctx.vars[prints[i]];
        os << (i ? "," : "") << "{\"fmt\":";
        json_string(os, *v.fmt);
        os << ",\"args\":[";
        for (int k = 0, n = 0; k < 3; ++k) if (v.dep[k]) os << (n++ ? "," : "") << v.dep[k];
        os << "],\"size\":" << v.size << "}";
    }
    os << "]}";
}

/* ------------------------------------------------------------------ launch */
/* the kernel arguments and grid of one sweep: allocates its outputs (jit.cu:1171-1174), passes the program and the
   literals in the kernel parameters or through the program cache, and fills in the data pointers */
bool sweep_args(EkContext &ctx, const Sweep &s, EkSweepArgs &args, uint32_t &grid, bool &inline_prog) {
    const Assembled &a = s.a;
    const Config &cfg = s.cfg;
    for (const Output &o : a.outputs) {
        EkVariable &v = ctx.vars[o.var];
        if (v.data == nullptr) { v.data = ek_malloc(o.bytes); v.free_data = true; v.subtree_size = 1; }
    }
    Program prog;
    if (!kernel_program(a, cfg, prog) || (cfg.fast && prog.size() > EK_INLINE_PROG)) {
        ek_set_error("ek_eval(): internal error: fast-kernel lowering failed after it had been checked"); return false;
    }
    memset(&args, 0, sizeof(args));
    inline_prog = prog.size() <= EK_INLINE_PROG;
    const bool inline_lit = a.lits.size() <= EK_MAX_LIT_INLINE;
    /* programs and literals that fit the kernel parameters travel there: nothing is uploaded and nothing is cached
       (a trace whose literals change from step to step -- a step counter, a learning-rate schedule -- used to add a
       cache entry and two synchronous uploads per step) */
    if (!inline_prog || !inline_lit) lookup_program(ctx, prog, a.lits, !inline_prog, !inline_lit, args.prog, args.lit);
    if (inline_prog) {
        EkInstr *dstp = args.prog_inline;
        for (const EkInstr &in : prog.init) *dstp++ = in;
        for (const EkInstr &in : prog.body) *dstp++ = in;
        for (const EkInstr &in : prog.fini) *dstp++ = in;
    }
    if (inline_lit && !a.lits.empty()) memcpy(args.lit_inline, a.lits.data(), a.lits.size() * 4);
    if (inline_lit) args.lit = nullptr;
    args.n_init = (uint32_t) prog.init.size(); args.n_body = (uint32_t) prog.body.size(); args.n_fini = (uint32_t) prog.fini.size();
    args.n_lit = (uint32_t) a.lits.size();
    args.n_argw = (uint32_t) a.argw.size();
    args.n_scalar = (uint32_t) a.scalars.size();
    args.n = (uint32_t) s.g->size;
    uint32_t tile = cfg.T * cfg.V;
    args.n_tiles = (uint32_t) ((s.g->size + tile - 1) / tile);
    args.n_tmp = a.n_tmp; args.n_in_units = a.n_in_units;
    args.n_staged = (uint32_t) a.staged.size();
    args.n_stages = cfg.stages;
    args.smem_bar_off = cfg.off_bar; args.smem_prog_off = cfg.off_prog;
    args.smem_extra_off = cfg.off_extra; args.smem_slots_off = cfg.off_slots;
    args.prog_in_smem = cfg.prog_in_smem ? 1 : 0;
    args.n_red = a.n_red;
    args.red_partials = ctx.red_partials; args.red_counters = ctx.red_counters;
    args.tma_ok = 1;
    for (size_t k = 0; k < a.staged.size(); ++k) {
        const EkVariable &v = ctx.vars[a.staged[k].var];
        if (v.data == nullptr) { ek_set_error("ek_eval(): internal error: staged input without data"); return false; }
        args.staged_ptr[k] = v.data;
        args.staged_unit[k] = a.staged[k].unit;
        args.staged_esize[k] = a.staged[k].esize;
        if (((uintptr_t) v.data & 15u) != 0) args.tma_ok = 0;
    }
    for (size_t k = 0; k < a.scalars.size(); ++k) {
        const EkVariable &v = ctx.vars[a.scalars[k].var];
        if (v.data == nullptr) { ek_set_error("ek_eval(): internal error: scalar input without data"); return false; }
        args.scalar_ptr[k] = v.data;
        args.scalar_type[k] = (uint8_t) v.type;
    }
    argument_words(a, cfg, args.argw);
    for (const auto &pf : a.ptr_fix) {
        uint64_t p = (uint64_t) (uintptr_t) ctx.vars[pf.var].data;
        args.argw[pf.argw] = (uint32_t) p; args.argw[pf.argw + 1] = (uint32_t) (p >> 32);
    }
    grid = std::min<uint32_t>(args.n_tiles, (uint32_t) ctx.num_sms * cfg.ctas_per_sm);
    grid = std::max(grid, 1u);
    if (grid > ctx.max_grid) grid = ctx.max_grid;
    return true;
}

bool launch_sweep(EkContext &ctx, const Sweep &s) {
    const Assembled &a = s.a;
    const Config &cfg = s.cfg;
    EkSweepArgs args; uint32_t grid; bool inline_prog;
    if (!sweep_args(ctx, s, args, grid, inline_prog)) return false;

    if (ctx.log_level >= 1)
        fprintf(stderr, "ek_eval(): launching sweep (n=%zu, in=%zu, out=%zu, ops=%u, slots=%u, V=%d, T=%u, stages=%u, grid=%u, smem=%zu)\n",
                s.g->size, a.staged.size() + a.scalars.size(), a.outputs.size(), a.n_arith, a.n_tmp, cfg.V, cfg.T, cfg.stages, grid, cfg.smem);
    if (ctx.log_level >= 3) { std::ostringstream oss; dump_program(oss, a, *s.g); fputs(oss.str().c_str(), stderr); }

    if (ctx.timing) ek_cuda_check(cudaEventRecord(ctx.ev_start, ctx.stream));
    if (cfg.fast) {
        ek_cuda_check(ek_launch_sweep_fast(args, grid, cfg.T, cfg.smem, ctx.stream));
    } else {
        bool trig = false;          /* the general kernel's instantiation with the trigonometric, hyperbolic, special, other math and Carlson operations */
        for (const EkInstr &in : a.body) trig |= ek_dop_ext(in.op);
        ek_cuda_check(ek_launch_sweep(cfg.V, inline_prog, trig, args, grid, cfg.T, cfg.smem, ctx.stream));
    }
    if (ctx.timing) {
        ek_cuda_check(cudaEventRecord(ctx.ev_stop, ctx.stream));
        ek_cuda_check(cudaEventSynchronize(ctx.ev_stop));
        float ms = 0; ek_cuda_check(cudaEventElapsedTime(&ms, ctx.ev_start, ctx.ev_stop));
        ctx.stats.last_kernel_ms = ms; ctx.stats.total_kernel_ms += ms;
    }
    ctx.stats.launches++; ctx.stats.sweep_launches++;
    if (cfg.fast) ctx.stats.fast_launches++;
    ctx.stats.ops_evaluated += (uint64_t) a.n_arith * s.g->size;
    ctx.stats.bytes_in += a.bytes_in; ctx.stats.bytes_out += a.bytes_out;
    return true;
}

/* ------------------------------------------------------------------ releasing the trace */
void clear_dirty(EkContext &ctx) {
    for (uint32_t idx : ctx.dirty) if (idx < ctx.vars.size()) ctx.vars[idx].dirty = false;
    ctx.dirty.clear();
}

/* clear the dependencies of `idx` and release the references they held */
void drop_deps(EkContext &ctx, uint32_t idx) {
    EkVariable &v = ctx.vars[idx];
    uint32_t deps[4] = { v.dep[0], v.dep[1], v.dep[2], v.dep[3] };
    uint32_t extra = v.extra_dep;
    v.dep[0] = v.dep[1] = v.dep[2] = v.dep[3] = 0; v.extra_dep = 0;
    for (int k = 0; k < 4; ++k) if (deps[k] >= EK_REG_RESERVED) {
        /* dec_ref_int without re-entrancy surprises: var table may shrink but indices stay valid (the last reference
           frees the variable through ek_dec_ref_ext) */
        EkVariable &d = ctx.vars[deps[k]];
        if (d.used && d.ref_int > 0) { if (--d.ref_int == 0 && d.ref_ext == 0) { d.ref_ext = 1; ek_dec_ref_ext(deps[k]); } }
    }
    if (extra >= EK_REG_RESERVED) ek_dec_ref_ext(extra);
}

/* a side effect has run: drop its dependencies and release the reference the trace held */
void retire_side_effect(EkContext &ctx, uint32_t idx) {
    EkVariable &v = ctx.vars[idx];
    v.side_effect = false;
    v.op = EK_OP_INVALID;
    drop_deps(ctx, idx);
    ek_dec_ref_ext(idx);
}

/* after the launches: drop the dependencies of everything that now has data (jit.cu:1484-1507), then retire the side
   effects that ran */
void retire(EkContext &ctx, const Schedule &s) {
    for (const Sweep &sw : s.sweeps) {
        for (uint32_t idx : sw.g->sched) {
            if (idx >= ctx.vars.size() || !ctx.vars[idx].used) continue;
            EkVariable &v = ctx.vars[idx];
            if (v.data != nullptr && v.op != EK_OP_INVALID && !v.direct_pointer) {
                v.op = EK_OP_INVALID;
                drop_deps(ctx, idx);
            }
        }
    }
    std::vector<uint32_t> side_effects;
    for (const Sweep &sw : s.sweeps) {
        for (uint32_t idx : sw.g->sched) {
            if (idx >= ctx.vars.size() || !ctx.vars[idx].used) continue;
            EkVariable &v = ctx.vars[idx];
            if (v.side_effect && v.op != EK_OP_INVALID) {
                if (std::find(side_effects.begin(), side_effects.end(), idx) == side_effects.end()) side_effects.push_back(idx);
            }
        }
    }
    for (uint32_t idx : side_effects) retire_side_effect(ctx, idx);
}

/* ------------------------------------------------------------------ prints (cuda_printf, jit.cu:863-916) */
/* where one printed argument's values come from */
struct PrintArg {
    uint32_t var = 0;
    ek_type type = EK_INVALID;
    size_t size = 1;
    bool immediate = false; uint64_t imm = 0;   /* literal / registered pointer: one value for every element */
    void *snapshot = nullptr;                   /* evaluated before this eval: its copy, taken before the first launch */
    std::vector<uint8_t> host;                  /* the values read back */
};
struct PrintJob { uint32_t node; std::vector<PrintArg> args; };

/* Before the first launch.  Arguments that are already evaluated are copied in stream order, so that a scatter of the
   same evaluation cannot change what is printed; computed arguments are stored by their sweeps (Planner::forced). */
std::vector<PrintJob> snapshot_prints(EkContext &ctx, const std::vector<uint32_t> &prints) {
    std::vector<PrintJob> jobs;
    for (uint32_t idx : prints) {
        PrintJob job; job.node = idx;
        for (int k = 0; k < 3; ++k) {
            uint32_t d = ctx.vars[idx].dep[k];
            if (d < EK_REG_RESERVED) continue;
            const EkVariable &dv = ctx.vars[d];
            PrintArg a; a.var = d; a.type = dv.type; a.size = dv.size;
            if (dv.direct_pointer) { a.immediate = true; a.imm = (uint64_t) (uintptr_t) dv.data; }
            else if (dv.data == nullptr && dv.op == EK_OP_LITERAL) { a.immediate = true; a.imm = dv.imm; }
            else if (dv.data != nullptr) {
                size_t bytes = dv.size * ek_type_size(dv.type);
                a.snapshot = ek_malloc(bytes);
                ek_cuda_check(cudaMemcpyAsync(a.snapshot, dv.data, bytes, cudaMemcpyDeviceToDevice, ctx.stream));
            }
            job.args.push_back(std::move(a));
        }
        jobs.push_back(std::move(job));
    }
    return jobs;
}

/* After the launches: one synchronisation, the read-back of every argument, then the lines of each print in recording
   order (elements ascending) on stdout, and one fflush. */
void run_prints(EkContext &ctx, std::vector<PrintJob> &jobs) {
    for (PrintJob &job : jobs)
        for (PrintArg &a : job.args) {
            if (a.immediate) continue;
            const void *src = a.snapshot ? a.snapshot : ctx.vars[a.var].data;
            if (!src) { fprintf(stderr, "ek_eval(): internal error: printed variable %u was not evaluated\n", a.var); exit(EXIT_FAILURE); }
            a.host.resize(a.size * ek_type_size(a.type));
            ek_cuda_check(cudaMemcpyAsync(a.host.data(), src, a.host.size(), cudaMemcpyDeviceToHost, ctx.stream));
        }
    ek_cuda_check(cudaStreamSynchronize(ctx.stream));
    std::string out;
    for (PrintJob &job : jobs) {
        for (PrintArg &a : job.args) { ek_free(a.snapshot); a.snapshot = nullptr; }
        const EkVariable &pv = ctx.vars[job.node];
        const uint32_t narg = (uint32_t) job.args.size();
        ek_type types[3] = { EK_INVALID, EK_INVALID, EK_INVALID };
        for (uint32_t k = 0; k < narg; ++k) types[k] = job.args[k].type;
        std::vector<EkPrintSeg> segs; std::string err;
        if (!ek_printf_parse(pv.fmt->c_str(), narg, types, segs, err)) {     /* (checked when it was recorded) */
            fprintf(stderr, "ek_eval(): internal error: %s\n", err.c_str()); exit(EXIT_FAILURE);
        }
        uint64_t bits[3] = { 0, 0, 0 };
        for (size_t i = 0; i < pv.size; ++i) {
            for (uint32_t k = 0; k < narg; ++k) {
                const PrintArg &a = job.args[k];
                if (a.immediate) { bits[k] = a.imm; continue; }
                const size_t es = ek_type_size(a.type);
                bits[k] = 0;
                memcpy(&bits[k], a.host.data() + (a.size == 1 ? 0 : i) * es, es);
            }
            ek_printf_append(out, segs, types, bits);
            if (out.size() >= ((size_t) 1 << 20)) { fwrite(out.data(), 1, out.size(), stdout); out.clear(); }
        }
    }
    fwrite(out.data(), 1, out.size(), stdout);
    fflush(stdout);
}

/* a print has run (or is discarded): free its format and release its arguments and the trace's reference */
void retire_prints(EkContext &ctx, const std::vector<uint32_t> &prints) {
    for (uint32_t idx : prints) {
        delete ctx.vars[idx].fmt; ctx.vars[idx].fmt = nullptr;
        retire_side_effect(ctx, idx);
    }
}

/* the prints of the dry runs: format, argument handles and size */
void dump_prints(std::ostream &os, const EkContext &ctx, const std::vector<uint32_t> &prints) {
    for (uint32_t idx : prints) {
        const EkVariable &v = ctx.vars[idx];
        os << "print n=" << v.size << " args=";
        for (int k = 0, n = 0; k < 3; ++k) if (v.dep[k]) os << (n++ ? "," : "") << v.dep[k];
        os << " fmt=";
        json_string(os, *v.fmt);
        os << "\n";
    }
}

} // namespace

/* ------------------------------------------------------------------ eval */
extern "C" {

int ek_eval(void) {
    ek_dlpack_drain();
    EkContext &ctx = ek_ctx();
    for (auto cb : ctx.callbacks) cb.first(cb.second);         /* jit.cu:1421-1422 */
    if (ctx.live.empty()) { clear_dirty(ctx); return 0; }
    if (ek_init() != 0) return -1;

    Schedule s(ctx);
    if (!s.build()) return -1;
    clear_dirty(ctx);                                          /* jit.cu:1430-1434 */
    ctx.live.clear();
    for (uint32_t idx : s.kept_literals) ctx.live.insert(idx);
    std::vector<PrintJob> jobs = snapshot_prints(ctx, s.prints);
    for (const Sweep &sw : s.sweeps)
        if (!launch_sweep(ctx, sw)) return -1;
    /* (only an evaluation that prints waits for its launches) */
    if (!jobs.empty()) run_prints(ctx, jobs);
    retire(ctx, s);
    retire_prints(ctx, s.prints);
    return 0;
}

int ek_eval_var(uint32_t index) {
    EkContext &ctx = ek_ctx();
    if (index < EK_REG_RESERVED || index >= ctx.vars.size() || !ctx.vars[index].used) {
        ek_set_error("ek_eval_var(): unknown variable " + std::to_string(index));
        return -1;
    }
    EkVariable &v = ctx.vars[index];
    if (v.data == nullptr && v.op == EK_OP_LITERAL) {
        /* literal: give it storage directly (no sweep needed) */
        if (ek_init() != 0) return -1;
        size_t es = ek_type_size(v.type);
        void *p = ek_malloc(v.size * es);
        ek_fill(p, es, v.imm, v.size);
        ctx.vars[index].data = p; ctx.vars[index].free_data = true; ctx.vars[index].op = EK_OP_INVALID;
        ctx.live.erase(index);
        return 0;
    }
    if (v.data == nullptr || v.dirty) return ek_eval();          /* jit.cu:1510-1515 */
    return 0;
}

/* host-only: assemble what ek_eval() would launch and return a textual listing (malloc'd).
   Used by the CPU test-suite to check scheduling / register allocation without a GPU. */
EK_API char *ek_debug_plan(void) {
    Schedule s(ek_ctx());
    if (!s.build()) return nullptr;
    std::ostringstream oss;
    for (const Sweep &sw : s.sweeps) dump_program(oss, sw.a, *sw.g);
    dump_prints(oss, ek_ctx(), s.prints);
    return strdup(oss.str().c_str());
}

/* host-only test aid: forget recorded scatters that can never run (CPU test-suite without a GPU), exactly as if they
   had been executed: the trace's own reference is released and the node leaves the live set */
EK_API void ek_debug_discard_side_effects(void) {
    EkContext &ctx = ek_ctx();
    std::vector<uint32_t> pending;
    for (uint32_t idx : ctx.live)
        if (idx < ctx.vars.size() && ctx.vars[idx].used && ctx.vars[idx].side_effect && ctx.vars[idx].op != EK_OP_INVALID) pending.push_back(idx);
    for (uint32_t idx : pending) { delete ctx.vars[idx].fmt; ctx.vars[idx].fmt = nullptr; retire_side_effect(ctx, idx); }
    clear_dirty(ctx);
}

/* same as ek_debug_plan(), as JSON with the complete programs (tests/ek_emulator.py); empty when nothing is live */
EK_API char *ek_debug_program(void) {
    EkContext &ctx = ek_ctx();
    Schedule s(ctx);
    if (!s.build()) return nullptr;
    std::ostringstream oss;
    if (!ctx.live.empty()) write_program_json(oss, ctx, s.sweeps, s.prints);
    return strdup(oss.str().c_str());
}

} /* extern "C" */
