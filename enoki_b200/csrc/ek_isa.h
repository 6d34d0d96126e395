/*
 * ek_isa.h -- device "sweep program" format shared by the host assembler
 * (ek_runtime.cpp) and the fused sweep kernel (ek_sweep.cu).
 *
 * The reference lowers the expression DAG to a PTX string per launch
 * (src/cuda/jit.cu:983-1227).  Here the DAG is lowered to a compact program of
 * 16-byte instructions executed by ONE hand-written sm_90a kernel; every
 * instruction processes V elements per thread with statically indexed registers,
 * values that must outlive the next instruction live in a shared-memory slot
 * file laid out [slot][group][thread] as 128-bit words.
 */
#pragma once
#include <stdint.h>

/* one instruction = 16 bytes.  Two-address accumulator machine: the first operand of every
   operation is the accumulator (the result of the previous instruction, held in registers),
   the others (b, c) are fetched from shared memory; the result replaces the accumulator and
   is additionally written to slot `dst` when EKF_ST is set. */
struct EkInstr {
    uint16_t op;      /* EkDop */
    uint16_t flags;
    uint16_t dst;     /* slot index for the result (if EKF_ST) / accumulator slot / uniform index */
    uint16_t b, c;    /* operand codes */
    uint16_t a;       /* operand loaded into the accumulator first (EKF_HAS_A) */
    uint32_t imm;
};

/* operand codes (16 bit) */
#define EK_OPND_NONE   0xFFFFu
#define EK_OPND_UNI    0x8000u          /* | word index into the (4x replicated) uniform pool        */
#define EK_OPND_STAGED 0x4000u          /* | slot unit inside the current pipeline stage (TMA input)   */
/* otherwise: temporary slot index */

/* flags */
#define EKF_ST    0x0001u   /* store the result to slot dst (dst+1 for the high plane)      */
#define EKF_R64   0x0002u   /* result is 64 bit (two planes)                                */
#define EKF_HAS_B 0x0004u
#define EKF_HAS_C 0x0008u
#define EKF_B64   0x0010u
#define EKF_C64   0x0020u
#define EKF_A64   0x0040u   /* the accumulator value is 64 bit (gather/scatter index, HAS_A)    */
#define EKF_HAS_A 0x0080u   /* load the accumulator from operand `a` before executing        */
#define EKF_NEG_A 0x0100u   /* f32 input modifier: accumulator = -accumulator                 */
#define EKF_ABS_A 0x0200u   /* f32 input modifier: accumulator = |accumulator|                */
#define EKF_RACC  0x4000u   /* after executing: fold the accumulator into the reduction partials in slot dst
                               (kind | class << 8 in field `a`; only when EKF_ST and EKF_HAS_A are clear)   */
#define EKF_STG   0x0400u   /* after executing, store the 32-bit accumulator to the global array
                               whose pointer is the uniform pair at index imm                 */

/* largest gather / scatter stride in bytes: it travels in the 15-bit field of imm (stride << 16); ek_trace_append
   refuses larger ones */
#define EK_MAX_GS_STRIDE 0x7fffu

/* rounding modes for DOP_CVT_* (imm) */
#define EK_RZ 0
#define EK_RM 1
#define EK_RP 2
#define EK_RN 3

/* reduction kinds */
#define EK_RED_SUM 0
#define EK_RED_PROD 1
#define EK_RED_MIN 2
#define EK_RED_MAX 3
/* reduction value classes */
#define EK_RC_F32 0
#define EK_RC_I32 1
#define EK_RC_U32 2
#define EK_RC_F64 3
#define EK_RC_I64 4
#define EK_RC_U64 5

/* R = accumulator, B / C = fetched operands.  Suffix R = reversed operand order (accumulator is
   the second operand), suffix C = accumulator is the addend of a fused multiply-add. */
#define EK_DOPS(X) \
    X(NOP) \
    /* f32 */ \
    X(ADD_F32) X(SUB_F32) X(SUBR_F32) X(MUL_F32) X(DIV_F32) X(DIVR_F32) X(FMA_F32) X(FMAC_F32) \
    X(MIN_F32) X(MINR_F32) X(MAX_F32) X(MAXR_F32) \
    X(ABS_F32) X(NEG_F32) X(SQRT_F32) X(RCP_F32) X(RSQRT_F32) \
    X(EXP_F32) X(LOG_F32) X(SIN_F32) X(COS_F32) \
    X(FLOOR_F32) X(CEIL_F32) X(ROUND_F32) X(TRUNC_F32) X(MULNZ_F32) X(FMANZ_F32) X(FMANZC_F32) \
    X(LT_F32) X(LE_F32) X(GT_F32) X(GE_F32) X(EQ_F32) X(NE_F32) \
    /* 32-bit integer */ \
    X(ADD_I32) X(SUB_I32) X(SUBR_I32) X(MUL_I32) X(MULHI_I32) X(MULHI_U32) \
    X(DIV_I32) X(DIVR_I32) X(DIV_U32) X(DIVR_U32) X(MOD_I32) X(MODR_I32) X(MOD_U32) X(MODR_U32) \
    X(MAD_I32) X(MADC_I32) X(MIN_I32) X(MIN_U32) X(MAX_I32) X(MAX_U32) \
    X(ABS_I32) X(NEG_I32) X(SHL_32) X(SHLR_32) X(SHR_I32) X(SHRR_I32) X(SHR_U32) X(SHRR_U32) \
    X(NOT_32) X(AND_32) X(OR_32) X(XOR_32) X(POPC_32) X(CLZ_32) X(CTZ_32) \
    X(LT_I32) X(LE_I32) X(GT_I32) X(GE_I32) X(LT_U32) X(LE_U32) X(GT_U32) X(GE_U32) X(EQ_32) X(NE_32) \
    X(NOT_B) X(SEXT8) X(SEXT16) X(ZEXT8) X(ZEXT16) X(NEZ_32) \
    /* f64 */ \
    X(ADD_F64) X(SUB_F64) X(SUBR_F64) X(MUL_F64) X(DIV_F64) X(DIVR_F64) X(FMA_F64) X(FMAC_F64) \
    X(MIN_F64) X(MINR_F64) X(MAX_F64) X(MAXR_F64) \
    X(ABS_F64) X(NEG_F64) X(SQRT_F64) X(RCP_F64) X(RSQRT_F64) \
    X(EXP_F64) X(LOG_F64) X(SIN_F64) X(COS_F64) \
    X(FLOOR_F64) X(CEIL_F64) X(ROUND_F64) X(TRUNC_F64) X(MULNZ_F64) X(FMANZ_F64) X(FMANZC_F64) \
    X(LT_F64) X(LE_F64) X(GT_F64) X(GE_F64) X(EQ_F64) X(NE_F64) \
    /* 64-bit integer */ \
    X(ADD_I64) X(SUB_I64) X(SUBR_I64) X(MUL_I64) X(MULHI_I64) X(MULHI_U64) \
    X(DIV_I64) X(DIVR_I64) X(DIV_U64) X(DIVR_U64) X(MOD_I64) X(MODR_I64) X(MOD_U64) X(MODR_U64) \
    X(MAD_I64) X(MADC_I64) X(MIN_I64) X(MIN_U64) X(MAX_I64) X(MAX_U64) \
    X(ABS_I64) X(NEG_I64) X(SHL_64) X(SHLR_64) X(SHR_I64) X(SHRR_I64) X(SHR_U64) X(SHRR_U64) \
    X(NOT_64) X(AND_64) X(OR_64) X(XOR_64) X(POPC_64) X(CLZ_64) X(CTZ_64) \
    X(LT_I64) X(LE_I64) X(GT_I64) X(GE_I64) X(LT_U64) X(LE_U64) X(GT_U64) X(GE_U64) X(EQ_64) X(NE_64) \
    /* select: _M accumulator is the mask (R = R ? B : C); _T accumulator is the true value \
       (R = B ? R : C, B = mask); _F accumulator is the false value (R = B ? C : R) */ \
    X(SEL_M_32) X(SEL_T_32) X(SEL_F_32) X(SEL_M_64) X(SEL_T_64) X(SEL_F_64) \
    /* accumulator loads / misc */ \
    X(LOAD_32) X(LOAD_64) X(INDEX) \
    /* conversions of the accumulator (imm = rounding mode for float->int) */ \
    X(CVT_F32_I32) X(CVT_F32_U32) X(CVT_I32_F32) X(CVT_U32_F32) \
    X(CVT_F32_F64) X(CVT_F64_F32) X(CVT_I32_F64) X(CVT_U32_F64) X(CVT_F64_I32) X(CVT_F64_U32) \
    X(CVT_F32_I64) X(CVT_F32_U64) X(CVT_F64_I64) X(CVT_F64_U64) \
    X(CVT_I64_F32) X(CVT_U64_F32) X(CVT_I64_F64) X(CVT_U64_F64) \
    X(CVT_I32_I64) X(CVT_U32_U64) X(CVT_64_32) \
    /* Float16 storage: f32 -> binary16 bits (round to nearest even), binary16 bits -> f32 (exact) */ \
    X(CVT_F32_F16) X(CVT_F16_F32) \
    /* staged-input unpack into the accumulator: b = staged operand code */ \
    X(LD_U8) X(LD_S8) X(LD_U16) X(LD_S16) X(LD_64) \
    /* direct (non-staged) loads into the accumulator: imm = uniform index of base pointer */ \
    X(LDG_32) X(LDG_64) X(LDG_U8) X(LDG_S8) X(LDG_U16) X(LDG_S16) \
    /* stores of the accumulator: imm = uniform index of base pointer */ \
    X(ST_32) X(ST_64) X(ST_8) X(ST_16) \
    /* gathers: index = accumulator, b = mask, imm = signed_index << 31 | stride << 16 | uniform index of base pointer */ \
    X(GATHER_32) X(GATHER_64) X(GATHER_U8) X(GATHER_S8) X(GATHER_U16) X(GATHER_S16) X(GATHER_32_SMEM) \
    /* scatters: index = accumulator, b = value, c = mask; imm as for gathers; accumulator unchanged */ \
    X(SCATTER_32) X(SCATTER_64) X(SCATTER_8) X(SCATTER_16) \
    X(SCATTER_ADD_F32) X(SCATTER_ADD_I32) X(SCATTER_ADD_F64) X(SCATTER_ADD_I64) \
    X(SCATTER_ADD_F32_SMEM) X(SCATTER_ADD_I32_SMEM) \
    /* reductions: RACC accumulates the accumulator into slot dst (imm = kind | class<<8); \
       RFIN: b = accumulator slot, dst = uniform index of result pointer, imm = kind|class<<8|red_index<<16 */ \
    X(RACC) X(RFIN) \
    /* init/fini helpers for privatised scatter_add bins and staged gather tables \
       (imm = descriptor index in the uniform pool; SMEM_ZERO: dst = 1 for float bins, which start at -0.0) */ \
    X(SMEM_ZERO) X(SMEM_LOAD_TABLE) X(SMEM_FLUSH_ADD_F32) X(SMEM_FLUSH_ADD_I32) \
    /* f32 trigonometric and hyperbolic functions of array_math.h and special functions of special.h (ek_math.cuh), \
       numbered last so that the operations above keep their numbers (ek_sweep_kernel<V, INLINE, false> carries none \
       of them: ek_dop_ext); ATAN2: R = y, B = x, ATAN2R: R = x, B = y */ \
    X(TAN_F32) X(COT_F32) X(ASIN_F32) X(ACOS_F32) X(ATAN_F32) X(ATAN2_F32) X(ATAN2R_F32) \
    X(SINH_F32) X(COSH_F32) X(TANH_F32) X(ASINH_F32) X(ACOSH_F32) X(ATANH_F32) X(CBRT_F32) \
    X(ERF_F32) X(ERFC_F32) X(ERFINV_F32) X(LGAMMA_F32) X(TGAMMA_F32) \
    /* further f32 functions of array_math.h and special.h; POW / HYPOT: R = x, B = y, POWR / HYPOTR: R = y, B = x */ \
    X(POW_F32) X(POWR_F32) X(FREXP_M_F32) X(FREXP_E_F32) X(HYPOT_F32) X(HYPOTR_F32) X(DAWSON_F32) X(ERFI_F32) \
    /* Carlson integrals of special.h; RF / RD: R = x, B = y, C = z; RC: R = x, B = y, RCR: R = y, B = x */ \
    X(CARLSON_RF_F32) X(CARLSON_RD_F32) X(CARLSON_RC_F32) X(CARLSON_RCR_F32)

enum EkDop : uint16_t {
#define X(n) DOP_##n,
    EK_DOPS(X)
#undef X
    DOP__COUNT
};

/* the operations that only the extension instantiations of the sweep kernels carry (ek_sweep_kernel<V, INLINE, true>;
   lowered, ek_fast_kernel<T, EK_FX_TRIG / EK_FX_HYP / EK_FX_SPEC / EK_FX_MATH / EK_FX_ELL>): tan ... carlson_rc, numbered after every other
   operation.  The imm field of these instructions is free, and a body that contains one runs on those instantiations. */
static inline bool ek_dop_ext(uint32_t op) { return op >= DOP_TAN_F32 && op < DOP__COUNT; }

/* ---- lowered instruction format of the 32-bit fast kernel (ek_sweep_fast.cu) ----
   The assembler's EkInstr stream is lowered once more at launch time (ek_eval.cpp: lower_fast): the fused accumulator
   load and the -x / |x| input modifiers become instructions of their own (the dispatch frame then never writes the
   accumulator, which is what lets ptxas keep it in one fixed register set), operand codes become absolute
   shared-memory offsets, and operations whose second operand is a literal / scalar pick a "_U" twin that reads ONE
   word from the uniform pool instead of staging 16 registers.
     x = fop | fflags << 16      y = b | c << 16      z = dst | aux << 16      w = imm
   b, c, dst: shared-memory byte offset >> 4 (per-thread operands: + 16 * tid, + 16 * T per 128-bit group), or a
   uniform-pool word index; aux: reduction kind | class << 8 (FF_RACC).  Same 16 bytes as EkInstr. */
#define FF_B    0x0001u   /* fetch per-thread operand B                                         */
#define FF_C    0x0002u   /* fetch per-thread operand C                                         */
#define FF_BU   0x0004u   /* broadcast uniform-pool word b into B (ops without a _U twin)       */
#define FF_CU   0x0008u   /* broadcast uniform-pool word c into C                               */
#define FF_ST   0x0010u   /* store the accumulator to slot dst                                  */
#define FF_STG  0x0020u   /* store the accumulator to the global array whose pointer is pool pair imm */
#define FF_RACC 0x0040u   /* fold the accumulator into the reduction partials in slot dst       */
#define FF_VU   0x0080u   /* scatters: the value operand is the uniform-pool word b             */
#define FF_MU   0x0100u   /* gathers / scatters: the mask operand is the uniform-pool word (b for gathers, c for scatters) */
#define FF_REL  0x0200u   /* (on a NOP) the staged inputs in imm (bit k: staged input k) are dead for this tile -- refill
                             their buffers with the CTA's next tile while the rest of the tile computes (early release) */
#define FF_POST (FF_ST | FF_STG | FF_RACC | FF_REL)   /* (one test per dispatch for everything after the operation) */

/* binary operations: every entry X has a twin X_U = X + 1 whose second operand is uniform-pool word b */
#define EK_FOPS2(X) \
    X(ADD_F32) X(SUB_F32) X(SUBR_F32) X(MUL_F32) X(DIV_F32) X(MIN_F32) X(MAX_F32) X(MULNZ_F32) \
    X(LT_F32) X(LE_F32) X(GT_F32) X(GE_F32) X(EQ_F32) X(NE_F32) \
    X(ADD_I32) X(SUB_I32) X(SUBR_I32) X(MUL_I32) X(MIN_I32) X(MIN_U32) X(MAX_I32) X(MAX_U32) \
    X(SHL_32) X(SHR_I32) X(SHR_U32) X(AND_32) X(OR_32) X(XOR_32) \
    X(LT_I32) X(LE_I32) X(GT_I32) X(GE_I32) X(LT_U32) X(LE_U32) X(GT_U32) X(GE_U32) X(EQ_32) X(NE_32)
/* everything else that may appear in a body */
#define EK_FOPS1(X) \
    X(FMA_F32) X(FMA_F32_UB) X(FMA_F32_UC) X(FMAC_F32) X(FMAC_F32_UB) \
    X(MAD_I32) X(MADC_I32) X(FMANZ_F32) X(FMANZC_F32) X(SEL_M_32) X(SEL_T_32) X(SEL_F_32) \
    X(ABS_F32) X(NEG_F32) X(SQRT_F32) X(RCP_F32) X(RSQRT_F32) X(EXP_F32) X(LOG_F32) X(SIN_F32) X(COS_F32) \
    X(EXPN_F32) X(SQRTA_F32)   /* exp(-x), sqrt(|x|): the input modifier folded into the operation */ \
    X(FLOOR_F32) X(CEIL_F32) X(ROUND_F32) X(TRUNC_F32) X(ABS_I32) X(NEG_I32) X(NOT_32) X(NOT_B) X(NEZ_32) \
    X(CVT_F32_I32) X(CVT_F32_U32) X(CVT_I32_F32) X(CVT_U32_F32) \
    X(LOAD) X(LOADU) X(INDEX) X(LD_U8) X(LD_S8) X(LDG_32) X(ST_32) X(ST_8) \
    X(GATHER_32) X(GATHER_32_SMEM) X(SCATTER_32) X(SCATTER_ADD_F32) X(SCATTER_ADD_I32) \
    X(SCATTER_ADD_F32_SMEM) X(SCATTER_ADD_I32_SMEM) X(RACC)
/* init / fini sections only (interpreted outside the hot loop) */
#define EK_FOPS0(X) \
    X(SMEM_ZERO) X(SMEM_LOAD_TABLE) X(SMEM_FLUSH_ADD_F32) X(SMEM_FLUSH_ADD_I32) X(RFIN)

/* Float16 storage, in the bodies that ek_fast16_kernel runs: LD_U16 + CVT_F16_F32 on a staged input, CVT_F32_F16 + ST_16
   of an output (numbered last, so that the operations of ek_fast_kernel keep their numbers) */
#define EK_FOPS16(X) X(LD_F16) X(ST_F16)

/* tan, cot, asin, acos, atan and atan2, in the bodies that the trig instantiations of ek_fast_kernel run (numbered after
   the Float16 operations).  ATAN2 / ATAN2R: the accumulator is y / x; _U: the other operand is uniform-pool word b */
#define EK_FOPST(X) X(TAN_F32) X(COT_F32) X(ASIN_F32) X(ACOS_F32) X(ATAN_F32) \
                    X(ATAN2_F32) X(ATAN2_F32_U) X(ATAN2R_F32) X(ATAN2R_F32_U)
/* sinh, cosh, tanh, asinh, acosh, atanh and cbrt, in the bodies that the hyp instantiations run (numbered last) */
#define EK_FOPSH(X) X(SINH_F32) X(COSH_F32) X(TANH_F32) X(ASINH_F32) X(ACOSH_F32) X(ATANH_F32) X(CBRT_F32)
/* erf, erfc, erfinv, lgamma and tgamma, in the bodies that the special-function instantiations run (numbered last) */
#define EK_FOPSS(X) X(ERF_F32) X(ERFC_F32) X(ERFINV_F32) X(LGAMMA_F32) X(TGAMMA_F32)
/* pow, frexp, hypot, dawson and erfi, in the bodies that the EK_FX_MATH instantiations run (numbered last).
   The binary ones: the accumulator is x (R forms: y); _UB = X + 1: the other operand is uniform-pool word b (as
   FMA_F32_UB) */
#define EK_FOPSM(X) X(POW_F32) X(POW_F32_UB) X(POWR_F32) X(POWR_F32_UB) X(FREXP_M_F32) X(FREXP_E_F32) \
                    X(HYPOT_F32) X(HYPOT_F32_UB) X(HYPOTR_F32) X(HYPOTR_F32_UB) X(DAWSON_F32) X(ERFI_F32)
/* carlson_rf, carlson_rd and carlson_rc, in the bodies that the EK_FX_ELL instantiations run (numbered last).  The
   accumulator is x (RCR: y); no uniform twins: a literal or scalar operand is broadcast (FF_BU / FF_CU) */
#define EK_FOPSE(X) X(CARLSON_RF_F32) X(CARLSON_RD_F32) X(CARLSON_RC_F32) X(CARLSON_RCR_F32)

/* feature bits of the ek_fast_kernel instantiations: the launcher runs the smallest one whose operations cover the
   lowered body */
#define EK_FX_F16  1u     /* FOP_LD_F16, FOP_ST_F16 */
#define EK_FX_TRIG 2u     /* EK_FOPST */
#define EK_FX_HYP  4u     /* EK_FOPSH */
#define EK_FX_SPEC 8u     /* EK_FOPSS */
#define EK_FX_MATH 16u    /* EK_FOPSM */
#define EK_FX_ELL  32u    /* EK_FOPSE */
#define EK_FX_ALL  (EK_FX_F16 | EK_FX_TRIG | EK_FX_HYP | EK_FX_SPEC | EK_FX_MATH | EK_FX_ELL)

enum EkFop : uint16_t {
    FOP_NOP,
#define X(n) FOP_##n, FOP_##n##_U,
    EK_FOPS2(X)
#undef X
#define X(n) FOP_##n,
    EK_FOPS1(X)
    EK_FOPS0(X)
    EK_FOPS16(X)
    EK_FOPST(X)
    EK_FOPSH(X)
    EK_FOPSS(X)
    EK_FOPSM(X)
    EK_FOPSE(X)
#undef X
    FOP__COUNT
};

/* the operation sets (EK_FX_*) that a lowered body uses: the instantiation of ek_fast_kernel that runs it */
static inline uint32_t ek_fast_ext(const EkInstr *body, uint32_t n) {
    uint32_t ext = 0;
    for (uint32_t pc = 0; pc < n; ++pc) {
        const uint32_t op = body[pc].op;
        if (op == FOP_LD_F16 || op == FOP_ST_F16) ext |= EK_FX_F16;
        else if (op >= FOP_CARLSON_RF_F32 && op < FOP__COUNT) ext |= EK_FX_ELL;
        else if (op >= FOP_POW_F32 && op <= FOP_ERFI_F32) ext |= EK_FX_MATH;
        else if (op >= FOP_ERF_F32 && op <= FOP_TGAMMA_F32) ext |= EK_FX_SPEC;
        else if (op >= FOP_SINH_F32 && op <= FOP_CBRT_F32) ext |= EK_FX_HYP;
        else if (op >= FOP_TAN_F32) ext |= EK_FX_TRIG;
    }
    return ext;
}

/* ---- launch arguments (passed by value as a __grid_constant__ kernel parameter) ---- */
#define EK_MAX_STAGED   16      /* staged (TMA) input arrays per sweep                  */
#define EK_MAX_ARGW     448     /* argument words appended to the uniform pool          */
#define EK_MAX_SCALAR   64      /* size-1 evaluated inputs fetched in the prologue      */
#define EK_MAX_LIT_INLINE 128   /* literal words carried inside the kernel parameters       */
#define EK_INLINE_PROG  448     /* instructions carried inside the kernel parameters (constant bank):
                                   instruction words are then uniform registers -> uniform branches */

struct EkSweepArgs {
    const EkInstr  *prog;          /* [n_init | n_body | n_fini] instructions (device memory; used when
                                      the program does not fit prog_inline)                   */
    const uint32_t *lit;           /* literal words (device memory, cached with the program); NULL: lit_inline */
    uint32_t n_init, n_body, n_fini;
    uint32_t n_lit;                /* literal words -> uniform pool [0, n_lit)               */
    uint32_t n_argw;               /* argument words -> uniform pool [n_lit, n_lit+n_argw)   */
    uint32_t n_scalar;             /* scalar inputs -> uniform pool (2 words each) after args */
    uint32_t n;                    /* number of elements                                      */
    uint32_t n_tiles;              /* ceil(n / tile)                                          */
    uint32_t n_tmp;                /* temporary slots                                         */
    uint32_t n_in_units;           /* slot units per pipeline stage                           */
    uint32_t n_staged;             /* staged input arrays                                     */
    uint32_t n_stages;             /* pipeline depth (2..4)                                   */
    uint32_t tma_ok;               /* all staged inputs 16-byte aligned                       */
    uint32_t smem_bar_off;         /* byte offsets inside dynamic shared memory:              */
    uint32_t smem_prog_off;        /*   mbarriers+reduction scratch, program copy,            */
    uint32_t smem_extra_off;       /*   privatised bins / staged tables,                      */
    uint32_t smem_slots_off;       /*   slot file (1024-byte aligned)                         */
    uint32_t prog_in_smem;         /* (global-memory programs) copy the program to shared memory */
    uint32_t n_red;                /* number of reductions                                    */
    uint64_t *red_partials;        /* [n_red][grid] 8-byte partials                           */
    uint32_t *red_counters;        /* [n_red] tickets (zero before and after the launch)      */
    const void *staged_ptr[EK_MAX_STAGED];
    uint16_t    staged_unit[EK_MAX_STAGED];   /* slot-unit offset inside a stage              */
    uint8_t     staged_esize[EK_MAX_STAGED];  /* 1, 2, 4 or 8                                 */
    const void *scalar_ptr[EK_MAX_SCALAR];
    uint8_t     scalar_type[EK_MAX_SCALAR];   /* ek_type                                      */
    uint32_t    argw[EK_MAX_ARGW];
    uint32_t    lit_inline[EK_MAX_LIT_INLINE]; /* literal words when they fit (nothing is uploaded, nothing is cached) */
    EkInstr     prog_inline[EK_INLINE_PROG];   /* valid when the launcher picks the INLINE kernel */
};
