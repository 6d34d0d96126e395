/*
 * enoki_b200.h -- C ABI of the H100-native backend for Enoki's two data-parallel
 * hot paths: the CUDAArray<T> expression-DAG evaluator and the DiffArray<T>
 * reverse-mode tape sweep.
 *
 * This is the drop-in boundary (SURVEY.md 8b): every entry point replaces one of
 * the C++-mangled `enoki::cuda_*` imports of the reference's libenoki-cuda.so
 * (declared in /root/reference/include/enoki/cuda.h:26-200) or one private
 * member of `enoki::Tape<CUDAArray<float>>` (include/enoki/autodiff.h:23-124,
 * defined in src/autodiff/autodiff.cpp).  The reference citation is given at
 * each declaration.  The single deliberate difference: the reference passes a
 * PTX *text* template to cuda_trace_append(); here the caller passes an opcode
 * (ek_op) -- the DAG is lowered to a small set of hand-written sm_90a kernels
 * instead of runtime-emitted PTX.
 *
 * Conventions
 *   - plain C types only; no C++/torch types cross this boundary.
 *   - variable handles are intrusively ref-counted uint32_t; 0 = "uninitialised"
 *     (cuda.h:954, jit.cu:43,287-290).
 *   - functions returning int return 0 on success and -1 on a *user* error
 *     (the conditions for which the reference throws std::runtime_error:
 *     jit.cu:207-212,366-371,386-388,722-725,777-782); functions returning a
 *     handle/pointer return 0/NULL on such an error.  ek_last_error() gives the
 *     message (thread-local, valid until the next call).  The C++ shim
 *     (include/enoki/cuda.h of this repo) rethrows std::runtime_error.
 *   - CUDA/driver failures and ref-count underflow print and exit(EXIT_FAILURE)
 *     exactly like the reference (common.cu:268-286, jit.cu:620-623).
 *   - single-threaded per process, one context per process (= per rank / GPU).
 */
#ifndef ENOKI_B200_H
#define ENOKI_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#  define EK_API
#else
#  define EK_API __attribute__((visibility("default")))
#endif

/* Same numbering as enoki::EnokiType (include/enoki/array_traits.h:522-524).  EK_FLOAT16 (IEEE binary16) is a storage
 * format: see ek_trace_append for what it accepts. */
typedef enum ek_type {
    EK_INVALID = 0, EK_INT8, EK_UINT8, EK_INT16, EK_UINT16, EK_INT32, EK_UINT32,
    EK_INT64, EK_UINT64, EK_FLOAT16, EK_FLOAT32, EK_FLOAT64, EK_BOOL, EK_POINTER
} ek_type;

/* Opcode vocabulary = SURVEY.md Appendix A (the PTX templates of
 * include/enoki/cuda.h:236-905 + the AD guards of autodiff.cpp:1198-1219). */
typedef enum ek_op {
    EK_OP_INVALID = 0,
    /* nullary */
    EK_OP_LITERAL,     /* cuda.h:267-317  mov.$t1 $r1, <imm>            (imm = raw bits) */
    EK_OP_INDEX,       /* cuda.h:641-663  mov.u32 $r1, $r2 (element index, UInt32)       */
    /* unary */
    EK_OP_MOV,         /* jit.cu:357-364  size-1 -> N broadcast copy                     */
    EK_OP_CVT,         /* cuda.h:236-247  cvt.rzi / cvt.rn / cvt                          */
    EK_OP_BITCAST,     /* cuda.h:249-258  mov.$b1                                         */
    EK_OP_NEG,         /* cuda.h:423-426 */
    EK_OP_ABS,         /* cuda.h:418-421 */
    EK_OP_SQRT,        /* cuda.h:428-431  sqrt.rn                                         */
    EK_OP_RCP,         /* cuda.h:459-462  (here: IEEE 1/x, see DESIGN.md numerics)        */
    EK_OP_RSQRT,       /* cuda.h:464-467 */
    EK_OP_EXP,         /* cuda.h:433-437  (here: Cephes exp of array_math.h:711-776)      */
    EK_OP_LOG,         /* cuda.h:439-443  (here: Cephes log of array_math.h:778-898)      */
    EK_OP_SIN,         /* cuda.h:445-448  (here: sincos_approx, array_math.h:261-367)     */
    EK_OP_COS,         /* cuda.h:450-453 */
    EK_OP_FLOOR,       /* cuda.h:469-472  cvt.rmi */
    EK_OP_CEIL,        /* cuda.h:474-477  cvt.rpi */
    EK_OP_ROUND,       /* cuda.h:479-482  cvt.rni */
    EK_OP_TRUNC,       /* cuda.h:484-487  cvt.rzi */
    EK_OP_FLOOR2INT,   /* cuda.h:489-492 */
    EK_OP_CEIL2INT,    /* cuda.h:494-497 */
    EK_OP_NOT,         /* cuda.h:525-528 */
    EK_OP_POPC,        /* cuda.h:530-533 */
    EK_OP_CLZ,         /* cuda.h:535-538 */
    EK_OP_CTZ,         /* cuda.h:540-543  brev+clz */
    /* binary */
    EK_OP_ADD,         /* cuda.h:341-348 */
    EK_OP_SUB,         /* cuda.h:350-357 */
    EK_OP_MUL,         /* cuda.h:359-366  mul.rn / mul.lo */
    EK_OP_MULHI,       /* cuda.h:368-371 */
    EK_OP_DIV,         /* cuda.h:373-380  div.rn / div */
    EK_OP_MOD,         /* cuda.h:382-385  rem */
    EK_OP_MIN,         /* cuda.h:413-416 */
    EK_OP_MAX,         /* cuda.h:408-411 */
    EK_OP_SHL,         /* cuda.h:499-506 */
    EK_OP_SHR,         /* cuda.h:508-517  arithmetic if signed */
    EK_OP_AND,         /* cuda.h:559-572  (value & mask when operand 2 is Bool)           */
    EK_OP_OR,          /* cuda.h:545-557 */
    EK_OP_XOR,         /* cuda.h:578-580 */
    EK_OP_GT,          /* cuda.h:582-588 */
    EK_OP_GE,          /* cuda.h:590-596 */
    EK_OP_LT,          /* cuda.h:598-604 */
    EK_OP_LE,          /* cuda.h:606-612 */
    EK_OP_EQ,          /* cuda.h:614-621 */
    EK_OP_NE,          /* cuda.h:623-630 */
    EK_OP_MUL_NZ,      /* autodiff.cpp:1191-1204 safe_mul:   (a==0||b==0) ? 0 : a*b       */
    /* ternary */
    EK_OP_FMA,         /* cuda.h:387-394  fma.rn / mad.lo */
    EK_OP_SELECT,      /* cuda.h:632-639  operands (mask, t, f) */
    EK_OP_FMA_NZ,      /* autodiff.cpp:1206-1221 safe_fmadd: (a==0||b==0) ? c : fma(a,b,c)*/
    /* memory; the target/source array is given by ek_set_scatter_gather_operand() and/or
       a Pointer variable (ek_var_register_ptr); `imm` = element stride in bytes          */
    EK_OP_GATHER,      /* cuda.h:845-864  operands (ptr, index, mask)                     */
    EK_OP_SCATTER,     /* cuda.h:866-890  operands (ptr, index, mask), value in `extra`   */
    EK_OP_SCATTER_ADD, /* cuda.h:892-905 */
    /* lazy horizontal reductions: result is a size-1 variable produced as an epilogue of
       the sweep that computes operand 1 (cuda.h:693-794 / horiz.cu:162-354 evaluate eagerly
       and re-read the operand with CUB; semantics identical)                              */
    EK_OP_HSUM, EK_OP_HPROD, EK_OP_HMAX, EK_OP_HMIN,
    EK_OP_ALL, EK_OP_ANY, EK_OP_COUNT,
    /* print node of ek_trace_printf() (jit.cu:863-916); not accepted by ek_trace_append()                  */
    EK_OP_PRINTF,
    /* Float32 only (other types are refused); appended so that no opcode above changes its number.  Each is ONE node
       that evaluates the single precision branch of array_math.h bit for bit as its traced form would              */
    EK_OP_TAN,         /* array_math.h:369-468  tancot_approx<true>                         */
    EK_OP_COT,         /* array_math.h:369-472  tancot_approx<false>                        */
    EK_OP_ASIN,        /* array_math.h:474-553 */
    EK_OP_ACOS,        /* array_math.h:555-601 */
    EK_OP_ATAN,        /* array_math.h:666-668  atan2(x, 1)                                 */
    EK_OP_ATAN2,       /* array_math.h:603-664  operands (y, x), like atan2(y, x)           */
    EK_OP_SINH,        /* array_math.h:997-1046 */
    EK_OP_COSH,        /* array_math.h:1048-1065 */
    EK_OP_TANH,        /* array_math.h:1129-1179 */
    EK_OP_ASINH,       /* array_math.h:1185-1237 */
    EK_OP_ACOSH,       /* array_math.h:1239-1293 */
    EK_OP_ATANH,       /* array_math.h:1295-1348 */
    EK_OP_CBRT,        /* array_math.h:900-954  frexp :682-709, ldexp :677-680              */
    EK_OP_ERF,         /* special.h:131-164 */
    EK_OP_ERFC,        /* special.h:56-129 */
    EK_OP_ERFINV,      /* special.h:222-246 */
    EK_OP_LGAMMA,      /* special.h:275-309 */
    EK_OP_TGAMMA,      /* special.h:312     exp(lgamma(x))                                  */
    EK_OP_POW,         /* array_math.h:956-958  exp(log(x) * y), operands (x, y)            */
    EK_OP_FREXP_M,     /* array_math.h:682-709  frexp(x).first: the mantissa                */
    EK_OP_FREXP_E,     /* array_math.h:682-709  frexp(x).second: the exponent, as a float   */
    EK_OP_HYPOT,       /* array_math.h:1362-1379  operands (a, b)                           */
    EK_OP_DAWSON,      /* special.h:249-265 */
    EK_OP_ERFI,        /* special.h:267-271  M_2_SQRTPI * dawson(x) * exp(x * x)            */
    EK_OP_CARLSON_RF,  /* special.h:325-366  carlson_rf(x, y, z), operands (x, y, z)         */
    EK_OP_CARLSON_RD,  /* special.h:379-432  carlson_rd(x, y, z), operands (x, y, z)         */
    EK_OP_CARLSON_RC,  /* special.h:445-482  carlson_rc(x, y), operands (x, y)               */
    EK_OP__COUNT
} ek_op;

/* ------------------------------------------------------------------ lifecycle */
EK_API int  ek_init(void);                 /* cuda.h:29  cuda_init      (jit.cu:274-318) */
EK_API void ek_shutdown(void);             /* cuda.h:32  cuda_shutdown  (jit.cu:320-326) */
EK_API const char *ek_last_error(void);    /* replaces thrown std::runtime_error::what() */
EK_API int  ek_device_count(void);         /* number of visible CUDA devices (0 on a CPU box, no error) */
EK_API int  ek_set_device(int ordinal);    /* new: one rank per GPU; must precede ek_init */
EK_API const char *ek_version(void);

/* ------------------------------------------------------------------ trace recording */
/* cuda.h:65-89 cuda_trace_append (4 arities).  a/b/c = operand handles (0 = unused),
 * imm = literal bits (EK_OP_LITERAL), rounding/stride payload, or the `value` operand
 * handle of SCATTER/SCATTER_ADD (4th operand).  Size/broadcast/dirty rules: jit.cu:701-861.
 * EK_FLOAT16 operands and results are accepted by LITERAL, MOV, CVT (through Float32, round to nearest even; not to Bool),
 * FLOOR2INT / CEIL2INT, BITCAST (to / from 16-bit integers), SELECT, GATHER and SCATTER; any other operation on them
 * is recorded but refused by the evaluation (ek_eval: an error naming Float16 -- convert to EK_FLOAT32 to compute). */
EK_API uint32_t ek_trace_append(ek_type type, ek_op op, uint32_t a, uint32_t b, uint32_t c,
                                uint64_t imm);
/* cuda.h:87-89 cuda_trace_printf (jit.cu:863-916): record a print of up to 3 arguments (any type but Float16).
 * Sizes, broadcast and errors as ek_trace_append (no arguments: size 1).  The format is checked now (ek_printf.cpp
 * lists what it may contain); a rejected format records nothing.  The evaluation that runs the print writes one
 * line per element to stdout, in recording order, before it returns, with each argument's value at recording time.
 * The library owns the node.  Returns 0, or -1 on a user error (ek_last_error()). */
EK_API int      ek_trace_printf(const char *fmt, uint32_t narg, const uint32_t *args);
EK_API void     ek_inc_ref_ext(uint32_t index);        /* cuda.h:41  (jit.cu:586-598) */
EK_API void     ek_dec_ref_ext(uint32_t index);        /* cuda.h:44  (jit.cu:614-638) */
EK_API size_t   ek_var_size(uint32_t index);           /* cuda.h:47 */
EK_API void    *ek_var_ptr(uint32_t index);            /* cuda.h:50  (NULL while unevaluated) */
EK_API ek_type  ek_var_type(uint32_t index);
EK_API uint32_t ek_var_set_size(uint32_t index, size_t size, int copy);  /* cuda.h:53 (jit.cu:339-371) */
EK_API int      ek_var_mark_dirty(uint32_t index);     /* cuda.h:56  (jit.cu:674-684) */
EK_API int      ek_var_set_label(uint32_t index, const char *label);     /* cuda.h:59 */
EK_API int      ek_var_mark_side_effect(uint32_t index);                 /* cuda.h:62 (jit.cu:663-672) */
EK_API int      ek_set_scatter_gather_operand(uint32_t index, int gather); /* cuda.h:65 (jit.cu:487-495) */
EK_API uint32_t ek_var_copy_to_device(ek_type type, size_t size, const void *host); /* cuda.h:131 (jit.cu:421-435) */
EK_API uint32_t ek_var_register_ptr(const void *ptr);  /* cuda.h:135 (jit.cu:397-419) */
EK_API uint32_t ek_var_register(ek_type type, size_t size, void *ptr, int dealloc); /* cuda.h:138 (jit.cu:373-395) */
EK_API int      ek_fetch_element(void *dst, uint32_t index, size_t offset, size_t size); /* cuda.h:142 (jit.cu:1520-1538) */
EK_API int      ek_make_managed(uint32_t index);       /* cuda.h:183 (jit.cu:455-485) */

/* ------------------------------------------------------------------ evaluation */
EK_API int  ek_eval(void);                             /* cuda.h:35  cuda_eval      (jit.cu:1418-1508) */
EK_API int  ek_eval_var(uint32_t index);               /* cuda.h:38  cuda_eval_var  (jit.cu:1510-1515) */
EK_API void ek_sync(void);                             /* cuda.h:177 cuda_sync */
EK_API int  ek_register_callback(void (*cb)(void *), void *payload);   /* cuda.h:186 */
EK_API int  ek_unregister_callback(void (*cb)(void *), void *payload); /* cuda.h:189 */
EK_API void     ek_set_log_level(uint32_t level);      /* cuda.h:195-200 */
EK_API uint32_t ek_log_level(void);
EK_API char    *ek_whos(void);                         /* cuda.h:180 (malloc'd; caller free()s) */

/* ------------------------------------------------------------------ eager horizontal ops on raw device memory
 * cuda.h:92-127 cuda_psum/hsum/hprod/hmax/hmin/count/compress/all/any/partition
 * (horiz.cu:35-354).  Results that are device pointers are owned by the caller
 * (release with ek_free) exactly like the reference.                                      */
EK_API void  *ek_hsum (ek_type type, size_t n, const void *data);
EK_API void  *ek_hprod(ek_type type, size_t n, const void *data);
EK_API void  *ek_hmax (ek_type type, size_t n, const void *data);
EK_API void  *ek_hmin (ek_type type, size_t n, const void *data);
EK_API void  *ek_psum (ek_type type, size_t n, const void *data);
EK_API size_t ek_count(size_t n, const uint8_t *mask);
EK_API int    ek_all  (size_t n, const uint8_t *mask);
EK_API int    ek_any  (size_t n, const uint8_t *mask);
EK_API int    ek_compress(ek_type type, size_t n, const void *data, const uint8_t *mask,
                          void **out_data, size_t *out_size);
EK_API int    ek_partition(size_t n, const void **ptrs, void ***unique_out,
                           uint32_t **counts_out, uint32_t ***perm_out);
EK_API void   ek_fill(void *ptr, size_t elem_size, uint64_t value, size_t n);   /* cuda.h:160-163 */
EK_API void   ek_reverse(void *out, const void *in, size_t elem_size, size_t n); /* cuda.h:166-169 */

/* ------------------------------------------------------------------ memory (jit.cu:1636-1896, common.cu:104-122) */
EK_API void *ek_malloc(size_t size);                   /* cuda.h:151 */
EK_API void *ek_managed_malloc(size_t size);           /* cuda.h:154 */
EK_API void *ek_host_malloc(size_t size);              /* cuda.h:157 */
EK_API void  ek_free(void *ptr);                       /* cuda.h:171 */
EK_API void  ek_host_free(void *ptr);                  /* cuda.h:174 */
EK_API void  ek_malloc_trim(void);                     /* cuda.h:177 */
EK_API void  ek_mem_get_info(size_t *free_bytes, size_t *total_bytes);  /* cuda.h:148 */
EK_API void  ek_memcpy_to_device(void *dst, const void *src, size_t size);         /* cuda.h:144 */
EK_API void  ek_memcpy_to_device_async(void *dst, const void *src, size_t size);
EK_API void  ek_memcpy_from_device(void *dst, const void *src, size_t size);       /* cuda.h:147 */
EK_API void  ek_memcpy_from_device_async(void *dst, const void *src, size_t size);
/* extension: device-to-host copy on the runtime's read-back stream (overlaps with later host-to-device copies and
   kernels; ordered after all work enqueued so far; keep `src` allocated until ek_sync()) */
EK_API void  ek_memcpy_from_device_overlapped(void *dst, const void *src, size_t size);
/* extension: device-to-device copy on the runtime's stream (PyTorch / CuPy interop, src/python/common.h:1085-1215) */
EK_API void  ek_memcpy_device_async(void *dst, const void *src, size_t size);

/* ------------------------------------------------------------------ DLPack (no counterpart in the reference)
 * Zero-copy exchange of device buffers with other frameworks (torch, CuPy, JAX).  The structures are in
 * enoki_b200_dlpack.h.  `versioned` selects DLManagedTensorVersioned (1) or the legacy DLManagedTensor (0).
 *
 * Export: evaluates the variable, takes an external reference on it and returns a managed tensor aliasing its buffer
 *   (kDLCUDA on ek_device(), 1-D shape {size}, strides NULL, byte_offset 0).  Float16/32/64 <-> kDLFloat, Int8..64 <->
 *   kDLInt, UInt8..64 <-> kDLUInt, Mask <-> kDLBool 8; pointer arrays are refused.  `consumer_stream` (a
 *   cudaStream_t, or NULL when the consumer declared none) is the stream the consumer uses the buffer on.  The
 *   tensor's deleter may run on any thread: it makes no runtime call, records an event on the consumer stream and
 *   queues the release; the owning thread makes the backend's stream wait on that event and drops the reference at
 *   its next entry into the runtime (ek_eval, ek_sync, ek_trace_append, ek_dlpack_*, ek_shutdown).
 * Import: returns a variable (reference count 1) that aliases the tensor and owns it.  Only kDLCUDA memory on
 *   ek_device(), lanes 1, the dtypes above and C-contiguous data (strides NULL or compact row-major, any ndim, any
 *   byte_offset aligned to the element) of 1 .. 2^32-1 elements are accepted; a versioned tensor must be of major
 *   version 1 and writable.  A refused tensor stays the caller's, and ek_last_error() names the reason; the checks
 *   make no CUDA call.  When the variable is freed, an event is recorded on the backend's stream and the producer's
 *   deleter is called once that event has completed (polled at later entries; ek_sync and ek_shutdown wait for it).
 *   The buffer never reaches the allocator: ek_free, its free lists and ek_malloc_trim never see it. */
EK_API void    *ek_dlpack_export(uint32_t index, int versioned, void *consumer_stream);
EK_API uint32_t ek_dlpack_import(void *managed, int versioned);
/* the CUDA device the backend runs on (the one ek_init() picks, before it has run) */
EK_API int      ek_device(void);
/* stream hand-off with a foreign cudaStream_t, one event record + stream wait each, no host synchronisation:
   ek_stream_wait_external: later work of the backend waits for what `stream` has enqueued so far;
   ek_stream_signal_external: later work on `stream` waits for what the backend has enqueued so far.
   Both initialise the backend; they return 0, or -1 when it cannot be (ek_last_error()). */
EK_API int      ek_stream_wait_external(void *stream);
EK_API int      ek_stream_signal_external(void *stream);

/* ------------------------------------------------------------------ reverse-mode tape
 * One tape per value type (Float32 / Float64) like the reference's static
 * Tape<CUDAArray<float>> / Tape<CUDAArray<double>> (autodiff.cpp:207-212,1235-1240).
 * Edge weights are evaluator variables (handles); gradients are returned as handles. */
EK_API uint32_t ek_tape_append_node(ek_type t, size_t size, const char *label);    /* autodiff.cpp:310-329 */
EK_API uint32_t ek_tape_append_leaf(ek_type t, size_t size);                        /* autodiff.cpp:331-338 */
EK_API int      ek_tape_append_edge(ek_type t, uint32_t src, uint32_t dst, uint32_t weight); /* autodiff.cpp:610-643 */
/* autodiff.cpp:266-308 append (1-3 inputs): returns 0 when all inputs are 0 */
EK_API uint32_t ek_tape_append(ek_type t, const char *label, size_t size, uint32_t n_in,
                               const uint32_t *in, const uint32_t *weights);
EK_API uint32_t ek_tape_append_gather(ek_type t, uint32_t offset_var, uint32_t mask_var);   /* autodiff.cpp:354-421 */
EK_API int      ek_tape_append_scatter(ek_type t, uint32_t src, uint32_t offset_var,
                                       uint32_t mask_var, int scatter_add);                  /* autodiff.cpp:523-608 */
EK_API uint32_t ek_tape_append_psum(ek_type t, uint32_t src);                                /* autodiff.cpp:470-521 */
EK_API uint32_t ek_tape_append_reverse(ek_type t, uint32_t src);                             /* autodiff.cpp:423-468 */
EK_API void     ek_tape_inc_ref_ext(ek_type t, uint32_t index);                              /* autodiff.cpp:726-736 */
EK_API void     ek_tape_dec_ref_ext(ek_type t, uint32_t index);                              /* autodiff.cpp:738-757 */
EK_API int      ek_tape_set_scatter_gather_operand(ek_type t, uint32_t *index, size_t size, int permute); /* autodiff.cpp:786-794 */
EK_API int      ek_tape_set_gradient(ek_type t, uint32_t index, uint32_t value_var, int backward); /* autodiff.cpp:822-836 */
EK_API int      ek_tape_backward(ek_type t, uint32_t index, int free_graph);                 /* autodiff.cpp:804-811,838-910 */
EK_API int      ek_tape_forward(ek_type t, uint32_t index, int free_graph);                  /* autodiff.cpp:813-820,912-988 */
EK_API int      ek_tape_backward_static(ek_type t, int free_graph);                          /* autodiff.cpp:838 */
EK_API int      ek_tape_forward_static(ek_type t, int free_graph);                           /* autodiff.cpp:912 */
EK_API uint32_t ek_tape_gradient(ek_type t, uint32_t index);   /* autodiff.cpp:796-802; borrowed handle (0 = none) */
EK_API int      ek_tape_set_label(ek_type t, uint32_t index, const char *label);             /* autodiff.cpp:340-352 */
EK_API void     ek_tape_push_prefix(ek_type t, const char *prefix);                          /* autodiff.cpp:776-778 */
EK_API int      ek_tape_pop_prefix(ek_type t);                                               /* autodiff.cpp:780-784 */
EK_API void     ek_tape_set_log_level(ek_type t, uint32_t level);                            /* autodiff.cpp:254-260 */
EK_API void     ek_tape_set_graph_simplification(ek_type t, int enable);                     /* autodiff.cpp:262-264 */
EK_API int      ek_tape_simplify(ek_type t);                                                 /* autodiff.cpp:990-1074 */
EK_API char    *ek_tape_graphviz(ek_type t, size_t n, const uint32_t *indices);              /* autodiff.cpp:1076-1163 (malloc'd) */
EK_API char    *ek_tape_whos(ek_type t);                                                     /* autodiff.cpp:1165-1189 (malloc'd) */
EK_API size_t   ek_tape_node_count(ek_type t);
EK_API void     ek_tape_clear(ek_type t);

/* ------------------------------------------------------------------ instrumentation (new; bench/tests) */
typedef struct ek_stats {
    uint64_t launches;          /* kernels of this library launched since the last reset */
    uint64_t sweep_launches;    /* ... of which fused evaluator sweeps                   */
    uint64_t adjoint_launches;  /* ... of which tape adjoint-level kernels               */
    uint64_t ops_evaluated;     /* array-ops: arithmetic DAG nodes x elements (jit.cu:1219-1222 `ops=`) */
    uint64_t edge_adjoints;     /* (edge, element) accumulations (autodiff.cpp:873-876)  */
    uint64_t bytes_in, bytes_out; /* algorithmic bytes streamed by sweeps (array loads / stores) */
    float    last_kernel_ms;    /* device time of the most recent timed launch (timing mode only) */
    float    total_kernel_ms;   /* sum of device times since reset (timing mode only)     */
    uint64_t fast_launches;     /* ... sweeps that ran on the 32-bit fast kernel (ek_sweep_fast.cu) */
    uint64_t partition_device;  /* ek_partition calls grouped on the device (the rest fell back to the host sort) */
} ek_stats;
/* ------------------------------------------------------------------ multi-GPU (SURVEY 8e; no counterpart in the reference)
 * One rank (process) per GPU, element-range sharding, ONE all-reduce of the size-1 results per step (the local hsum is
 * where the reference has it, autodiff.cpp:867-871).  NCCL is dlopen()ed on first use (EK_NCCL_LIB, else libnccl.so.2).
 * Rank 0: ek_dist_unique_id() -> hand the EK_DIST_ID_BYTES bytes to the other ranks; all ranks: ek_dist_init(). */
#define EK_DIST_ID_BYTES 128
EK_API int  ek_dist_unique_id(void *out_id);                         /* ncclGetUniqueId */
EK_API int  ek_dist_init(int rank, int world, const void *id);       /* ncclCommInitRank on the device of ek_set_device() */
EK_API int  ek_dist_rank(void);
EK_API int  ek_dist_world(void);
EK_API int  ek_allreduce(ek_type type, void *data, size_t count);    /* in-place sum on the backend's stream */
EK_API int  ek_allreduce_scalars(const uint32_t *handles, size_t n); /* evaluate + sum the given variables over all ranks */
EK_API void ek_dist_shutdown(void);

/* 32-bit fast sweep kernel (no counterpart in the reference): on by default; these calls read / override that
   (0 = general kernels only). */
EK_API void ek_set_fast_mode(int enable);
EK_API int  ek_fast_mode(void);
EK_API void ek_stats_reset(void);
EK_API void ek_stats_get(ek_stats *out);
EK_API void ek_set_timing(int enable);     /* bracket every launch with CUDA events on the launch stream */
EK_API void *ek_stream(void);              /* the cudaStream_t all kernels are launched on */
/* device timer on the launch stream: returns milliseconds between start and stop */
EK_API void  ek_timer_start(void);
EK_API float ek_timer_stop(void);
/* write `bytes` (>= L2 size) to a scratch buffer to flush L2 between timed iterations */
EK_API void  ek_flush_l2(void);

#ifdef __cplusplus
}
#endif
#endif /* ENOKI_B200_H */
