"""GPU: every 32-bit and narrow-integer element-wise operation on both sweep kernels, against exact references.

Types: Float32, Int32, UInt32 (the fast kernel's types) and Int8, UInt8, Int16, UInt16 (staged narrow inputs, 32-bit
arithmetic, narrowed results, narrow stores; only 8-bit comparisons, selects and bit operations have fast forms; every narrow result is also read
back as a 32-bit copy of its register, which must hold it sign- or zero-extended).  Operands: every pair of a table of
edge values (tests/test_gpu_conversions.py `F32_EDGES`, `_int_edges`, `shift_counts`) plus random values over all exponents / bit
lengths.  References, bit for bit (NaN matches NaN), no ulp tolerance:
  - Float32: numpy float32 for + - * / sqrt floor ceil rint trunc and the comparisons; 1 / x and 1 / sqrt(x) in
    float32 (rcp; rsqrt rounds twice, like RSQRT_F32); fma rounded once from fractions.Fraction; mul_nz / fma_nz
    (+0 / the addend when a factor is 0); min / max `a < b ? a : b` / `a > b ? a : b` (the second operand for NaN and
    for +-0 ties, DESIGN.md 4); exp / log / sin / cos from the C oracle (or_unary_f32); select, x & mask, x | mask
    as bit selects;
  - integers: Python integers wrapped to the type, with the kernels' pinned rules where the reference is undefined
    (division and modulo by 0, MIN / -1, shift counts of 32 or more) and the narrow bit counts counting the 32-bit
    sign- or zero-extended value (DESIGN.md 4).
Forms: every operand position of a binary / ternary operation in the accumulator (the reversed and swapped opcodes are
asserted from the plan), and a literal / an evaluated size-1 array in each position with the other operands loaded or
in the accumulator.  Each case runs on the fast and on the general kernel (`hz.kernel`) at sizes 1, 4097 and 2^20 + 7;
the variants the fast kernel has no operation for (integer mulhi / div / mod / bit counts, DIVR / MINR / MAXR_F32, the
reversed integer shifts, narrow arithmetic) are evaluated in programs of their own, which must not run on it, so
that they never take the other variants off it.  In the fast-mode runs the test asserts from the dry run
(ek.debug_program()) that the fast kernel's own forms occur in the bodies it runs: every _U twin, FMA_F32_UB / _UC,
FMAC_F32_UB (with the operand swap of a uniform C), the FF_BU / FF_CU broadcasts of MAD_I32, FMANZ_F32 and the selects,
EXPN_F32 and SQRTA_F32.  At 2^20 + 7 the Float32 rows come in blocks of 4096 whose values are all, none or partly in
the range of sqrt's MUFU.RSQ path, and `test_sqrt_every_input` runs sqrt on all 2^32 Float32 inputs.

tests/test_cpu_ops32.py runs the same cases through the planner, the assembler, the sweep-ISA emulator and the fast
kernel's source compiled for the host."""
import ctypes
import time

import numpy as np
import pytest

import test_gpu_conversions as cv
import test_gpu_gather_scatter as gs
import test_gpu_horizontal as hz

pytestmark = pytest.mark.gpu

TYPES = ("Float32", "Int32", "UInt32", "Int8", "UInt8", "Int16", "UInt16")
FAST_TYPES = ("Float32", "Int32", "UInt32")
SIZES = [1, 4097, (1 << 20) + 7]
FORMS = ("array", "literal", "scalar")
F32_OPS = list(cv.FLOAT_OPS) + list(cv.F32_ONLY) + ["expn", "sqrta"] + list(cv.MASK_OPS)
INT_OPS = list(cv.INT_OPS) + ["shl", "shr", "and_mask", "or_mask"]
MAX_CHECKS = 40                  # checks per evaluated program (the fast kernel takes bodies of <= 448 instructions)


def ops_of(tname, form):
    table = F32_OPS if tname == "Float32" else INT_OPS
    return [op for op in table if form == "array" or cv.arity(tname, op) > 1]


def variants(tname, op, form):
    """(position of the single value or None, variant) of each check group ops_case builds for op."""
    ar = cv.arity(tname, op)
    if form == "array":
        return [(None, f"acc{k}") for k in range(ar)]
    if ar == 1:
        return []
    return [(pos, var) for pos in range(ar) for var in ["plain"] + [f"acc{k}" for k in range(ar) if k != pos]]


def checks_of(tname, op, form):
    per = 2 if tname in cv.WIDE_OF else 1              # (a narrow result is checked twice: narrow and as 32 bits)
    if form == "array":
        return per * len(variants(tname, op, form))
    n = 0
    for pos, _ in variants(tname, op, form):
        n += 2 if cv.operand_types(tname, op)[pos] == "Bool" else len(cv.literal_values(tname, op, [0]))
    return per * n


def general_only(tname, op, pos, variant):
    """Whether the fast kernel lacks the operation this variant lowers to (the program then runs on the general
    kernel)."""
    if tname not in FAST_TYPES:
        # narrow arithmetic ends in SEXT8 / ZEXT8 / SEXT16 / ZEXT16 and 16-bit inputs load with LD_S16 / LD_U16: only
        # the operations that need no narrowing (comparisons, selects, and / or / xor with masks or values, so also
        # the x ^ 0 copies) of staged 8-bit inputs (LD_S8 / LD_U8) have fast forms
        return not (cv.WIDTH[tname] == 8 and op in cv.COMPARE + ("and", "or", "xor") + cv.MASK_OPS)
    acc1 = variant == "acc1"
    if tname == "Float32":
        return op in ("div", "min", "max") and acc1   # DIVR_F32, MINR_F32, MAXR_F32
    if op in ("mulhi", "div", "mod", "popc", "clz", "ctz"):
        return True
    return op in ("shl", "shr") and acc1              # SHLR_32, SHRR_I32, SHRR_U32


def programs_of(tname, form):
    """[(ops, keep, on_fast)]: the evaluations of one (type, form), each at most MAX_CHECKS checks, the variants the fast
    kernel has no operation for in programs of their own."""
    out = []
    for on_fast in (True, False):
        keep = (lambda op, pos, var, f=on_fast: general_only(tname, op, pos, var) != f)
        chunk, size = [], 0
        for op in ops_of(tname, form):
            k = sum(1 for pos, var in variants(tname, op, form) if keep(op, pos, var))
            if not k:
                continue
            k = checks_of(tname, op, form) * k // len(variants(tname, op, form))
            if chunk and size + k > MAX_CHECKS:
                out.append((chunk, keep, on_fast))
                chunk, size = [], 0
            chunk.append(op)
            size += k
        if chunk:
            out.append((chunk, keep, on_fast))
    return out


# ------------------------------------------------------------------ the fast kernel's own forms
def fast_bodies(programs):
    """(fop name, flags) of every lowered instruction in the bodies that run on the fast kernel, and the assembled
    instructions (op name, flags, dst, b, c, a, imm) of those sweeps."""
    lowered, assembled = [], []
    for prog in programs:
        for sw in prog["sweeps"]:
            if sw["config"]["fast"] and "fast" in sw:
                lowered += [(prog["fops"][t[0]], t[1]) for t in sw["fast"]["body"]]
                assembled += [(prog["ops"][t[0]],) + tuple(t[1:]) for t in sw["body"]]
    return lowered, assembled


FF_BU, FF_CU = 0x4, 0x8
UNI = 0x8000


def required_forms(tname, form, fops):
    """The fast kernel's forms a (type, form) must reach: names, or (name, flag) for a broadcast operand."""
    if tname not in FAST_TYPES:
        return set()
    if form == "array":
        return {"EXPN_F32", "SQRTA_F32"} if tname == "Float32" else set()
    twins = [f for f in fops if f.endswith("_U") and f[:-2] in fops and not f.startswith("ATAN2")]
    if tname == "Float32":
        req = {f for f in twins if f.endswith("_F32_U")}
        req |= {"FMA_F32_UB", "FMA_F32_UC", "FMAC_F32_UB", ("FMANZ_F32", FF_BU), ("FMANZ_F32", FF_CU)}
    elif tname == "Int32":
        req = {f for f in twins if f.endswith(("_I32_U", "_32_U"))} | {("MAD_I32", FF_BU), ("MAD_I32", FF_CU)}
    else:
        req = {f for f in twins if f.endswith(("_U32_U", "_32_U"))}
        req |= {"ADD_I32_U", "SUB_I32_U", "SUBR_I32_U", "MUL_I32_U", ("MAD_I32", FF_BU), ("MAD_I32", FF_CU)}
    return req | {("SEL", FF_BU), ("SEL", FF_CU)}


def check_fast_forms(tname, form, programs):
    lowered, assembled = fast_bodies(programs)
    fops = programs[0]["fops"]
    present = {name for name, _ in lowered}
    for name, fl in lowered:
        for bit in (FF_BU, FF_CU):
            if fl & bit:
                present.add((name, bit))
                if name.startswith("SEL_"):
                    present.add(("SEL", bit))
    missing = sorted(map(str, required_forms(tname, form, fops) - present))
    assert not missing, f"fast forms missing from the lowered bodies: {missing}"
    if tname == "Float32" and form != "array":
        # FMAC_F32 with only C uniform: lower_fast swaps B and C into FMAC_F32_UB
        assert any(op == "FMAC_F32" and c != 0xffff and c & UNI and not b & UNI for op, _fl, _d, b, c, *_ in assembled), \
            "no FMAC_F32 with a uniform C only"


# ------------------------------------------------------------------ tests
PARAMS = [(t, f, m) for t in TYPES for f in FORMS for m in ("fast", "general")]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("tname,form,mode", PARAMS)
def test_ops32(gpu, oracle, tname, form, mode, n):
    programs = []
    for k, (ops, keep, on_fast) in enumerate(programs_of(tname, form)):
        # (fast mode: a program of the fast kernel's operations must run on it once it is wide; the others never may)
        expect = None if mode != "fast" else (True if n > 4096 else None) if on_fast else False
        build = lambda put: cv.ops_case(gpu, put, tname, ops, n, form, seed=n + 31 * k, keep=keep, oracle=oracle)
        cv.run(gpu, build, mode, expect, programs if expect else None)
    if mode == "fast" and n > 4096 and tname in FAST_TYPES:
        check_fast_forms(tname, form, programs)


REF_UNARY = ("sqrt", "floor", "ceil", "round", "trunc", "abs", "neg", "exp", "log", "sin", "cos")
REF_BINARY = ("add", "sub", "mul", "div", "min", "max")


@pytest.mark.parametrize("mode", ["fast", "general"])
def test_f32_matches_the_reference_cpu_path(gpu, ref, mode):
    """DESIGN.md 4's "bit-identical to the reference" on the edge vectors: the kernels' Float32 results against the
    reference CPU path (oracle/_ref/libenoki_ref.so).  min / max are compared where no operand is NaN and the operands
    differ: the reference returns its first operand for NaN and for +-0 ties, this backend its second."""
    if ref is None:
        pytest.skip("the reference CPU path (oracle/_ref/libenoki_ref.so) is not built")
    rng = np.random.default_rng(77)
    a, b, c = (np.array(v, np.float64).astype(np.float32) for v in cv.float_operands("Float32", 700, rng))
    n = max(len(a), 4097)
    idx = np.arange(n) % len(a)
    a, b, c = a[idx], b[idx], c[idx]
    P = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    with hz.kernel(gpu, mode):
        A, B, C = (gpu.Float32.copy(x) for x in (a, b, c))
        got = {op: cv.apply(gpu, op, A) for op in REF_UNARY}
        got.update({op: cv.apply(gpu, op, A, B) for op in REF_BINARY})
        got["fma"] = cv.apply(gpu, "fma", A, B, C)
        gpu.lib().ek_stats_reset()
        gpu.cuda_eval()
        assert (gpu.stats().fast_launches >= 1) == (mode == "fast")
        bad = []
        for op, var in got.items():
            want = np.zeros(n, np.float32)
            if op == "fma":
                ref.ref_fmadd_f32(P(a), P(b), P(c), P(want), ctypes.c_size_t(n))
            elif op in REF_BINARY:
                assert ref.ref_binary_f32(op.encode(), P(a), P(b), P(want), ctypes.c_size_t(n)) == 0
            else:
                assert ref.ref_unary_f32(op.encode(), P(a), P(want), ctypes.c_size_t(n)) == 0
            g = var.numpy()
            ok = (g.view(np.uint32) == want.view(np.uint32)) | (np.isnan(g) & np.isnan(want))
            if op in ("min", "max"):
                ok |= np.isnan(a) | np.isnan(b) | (a == b)
            if not ok.all():
                k = int(np.flatnonzero(~ok)[0])
                bad.append(f"{op}: {int((~ok).sum())} differ, first a={a[k]!r} b={b[k]!r}: got {g[k]!r}, ref {want[k]!r}")
        assert not bad, "; ".join(bad)


CHUNK = 1 << 28


def test_sqrt_every_input(gpu):
    """sqrt on every Float32 bit pattern, on both kernels, and sqrt(|x|) (SQRTA_F32) on the fast kernel, in chunks of
    2^28 inputs generated on the device, against numpy's correctly rounded float32 sqrt.  The negative half reuses the
    positive half's reference: sqrt(-x) is NaN (-0 for -0) and sqrt(|-x|) = sqrt(x)."""
    ek = gpu
    t0 = time.perf_counter()

    def device(offset, fn, mode):
        with hz.kernel(ek, mode):
            x = ek.reinterpret(ek.Float32, ek.UInt32.arange(CHUNK) + np.uint32(offset))
            y = fn(x)
            ek.lib().ek_stats_reset()
            ek.cuda_eval()
            fast = ek.stats().fast_launches
            got = y.numpy().view(np.uint32)
        assert (fast >= 1) == (mode == "fast"), (mode, fast)
        return got

    def compare(label, got, want):
        bad = got != want.view(np.uint32)
        if bad.any():
            k = np.flatnonzero(bad)
            nan = np.isnan(got[k].view(np.float32)) & np.isnan(want[k])
            k = k[~nan]
            assert k.size == 0, f"{label}: {k.size} wrong, first input 0x{int(offset + k[0]) & 0xffffffff:08x}: " \
                                f"got 0x{int(got[k[0]]):08x}, want 0x{int(want.view(np.uint32)[k[0]]):08x}"

    for offset in range(0, 1 << 31, CHUNK):
        x = np.arange(offset, offset + CHUNK, dtype=np.uint32).view(np.float32)
        want = np.sqrt(x)
        del x
        neg = np.full(CHUNK, np.nan, np.float32)
        if offset == 0:
            neg[0] = -0.0
        for mode in ("fast", "general"):
            compare(f"sqrt {mode}", device(offset, ek.sqrt, mode), want)
        compare("sqrt(|x|) fast", device(offset, lambda v: ek.sqrt(abs(v)), "fast"), want)
        offset |= 1 << 31
        for mode in ("fast", "general"):
            compare(f"sqrt {mode}", device(offset, ek.sqrt, mode), neg)
        compare("sqrt(|x|) fast", device(offset, lambda v: ek.sqrt(abs(v)), "fast"), want)
    print(f"sqrt of every input: {time.perf_counter() - t0:.1f} s")
