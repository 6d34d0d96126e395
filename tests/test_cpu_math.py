"""CPU: the Float32 operations pow, frexp, hypot, dawson and erfi (EK_OP_POW ... EK_OP_ERFI).  What the
planner records and lowers for them (ek_debug_program): one operation each, their uniform-operand (_UB) and reversed
forms, Float16 storage around them; the operations it refuses; the C restatements of tests/math_oracle.c against the
reference CPU path (tests/golden/math.npz) and against the traced bodies they replace (tests/golden/math_traced.json,
run on the numpy interpreter); random expression DAGs that contain them on the numpy interpreter and on the
host-compiled fast kernel (tests/cpu_kernel), bit for bit; and the SASS of the kernels that carry them and of those that
must not change."""
import gc
import hashlib
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import math_support as ms
from ek_emulator import Emulator
from fast_kernel_emu import FastKernelEmulator
from test_cpu_emulator import _Factory

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CSRC = os.path.join(ROOT, "enoki_b200", "csrc")
BINARY, UNARY = ms.BINARY, ms.UNARY
# the number of body instructions of the traced bodies (one sweep each: the dry run stored in
# tests/golden/math_traced.json; frexp has two outputs)
TRACED = {"pow": 3, "frexp": 13, "hypot": 16, "dawson": 20, "erfi": 24}
MATH_EXT = 16


@pytest.fixture(autouse=True)
def clean_trace(ek):
    gc.collect()
    ek.lib().ek_debug_discard_side_effects()
    gc.collect()
    yield
    gc.collect()
    ek.lib().ek_debug_discard_side_effects()
    gc.collect()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _golden():
    return np.load(os.path.join(GOLDEN, "math.npz"))


def _traced():
    with open(os.path.join(GOLDEN, "math_traced.json")) as f:
        return json.load(f)


def _call(ek, name, *args):
    if name in ("frexp_m", "frexp_e"):
        return ek.frexp(*args)[name == "frexp_e"]
    return getattr(ek, {"pow": "pow_"}.get(name, name))(*args)


# ------------------------------------------------------------------ the C restatements against the reference CPU path
@pytest.mark.parametrize("name", BINARY + UNARY)
def test_restatement_against_math_golden(name):
    """raw bits, NaN payloads apart (x86 propagates the first NaN operand's, and the recorded program and the CPU path
    do not always meet the NaNs in the same order)"""
    d = _golden()
    args = (d["bx"], d["by"]) if name in BINARY else (d["x"],)
    got, want = ms.call(name, *args), d[name]
    bad = ~ms.same_bits(got, want)
    assert not bad.any(), (name, [a[bad][:5] for a in args], got[bad][:5], want[bad][:5])


def test_reference_edge_values_are_reproduced():
    """What array_math.h and special.h compute at their edges, reproduced as it is: pow(0, 0) = exp(-inf * 0) is NaN,
    pow of a negative base is NaN (log of it is), pow(0, y > 0) is 0, pow(inf, y > 0) inf and pow(1, inf) NaN (0 * inf);
    frexp treats denormals as normal numbers (mantissa with its leading zeros, exponent
    -127) and returns (x, 0) for 0, inf and NaN; hypot(inf, NaN) is inf + NaN = NaN.  The reference CPU path gives the
    same values."""
    inf, nan = np.inf, np.nan
    b = lambda u: np.array([u], np.uint32).view(np.float32)[0]
    cases = {
        "pow": ([(0.0, 0.0), (-2.0, 2.0), (0.0, 2.0), (inf, 0.5), (2.0, 0.5), (1.0, inf), (4.0, -0.5)],
                [nan, nan, 0.0, inf, 1.4142135, nan, 0.5]),
        "hypot": ([(3.0, 4.0), (inf, nan), (0.0, 0.0), (-0.0, -0.0), (1e30, 1e30), (nan, 1.0)],
                  [5.0, nan, 0.0, 0.0, 1.4142135e30, nan]),
    }
    for name, (pairs, wants) in cases.items():
        x = np.array([p[0] for p in pairs], np.float32); y = np.array([p[1] for p in pairs], np.float32)
        got = ms.binary(name, x, y)
        for xv, yv, g, w in zip(x, y, got, wants):
            if w is not None:
                assert ms.same_bits(g, np.float32(w)), (name, xv, yv, g, w)
    x = np.array([b(1), b(0x007fffff), 0.0, -0.0, inf, -inf, nan, 3.0, -0.75], np.float32)
    m, e = ms.unary("frexp_m", x), ms.unary("frexp_e", x)
    assert list(_bits(m[:2])) == [0x3f000001, 0x3f7fffff]
    assert list(e[:2]) == [-127, -127]
    assert ms.same_bits(m[2:7], x[2:7]).all() and (e[2:7] == 0).all()
    assert list(m[7:]) == [0.75, -0.75] and list(e[7:]) == [1, -1]
    # the same values on the CPU path
    d = _golden()
    for name in BINARY:
        k = np.flatnonzero((_bits(d["bx"]) == _bits(np.float32(0.0))) & (_bits(d["by"]) == _bits(np.float32(0.0))))
        assert len(k)
        assert ms.same_bits(d[name][k[0]], ms.binary(name, [0.0], [0.0])[0]), name


# ------------------------------------------------------------------ the restatements are the traced bodies
def _inputs(n, seed, name):
    """random bit patterns, then values over the ranges where the functions are used"""
    rng = np.random.default_rng(seed)
    r = rng.integers(0, 1 << 32, (2, n), dtype=np.uint64).astype(np.uint32).view(np.float32)
    q = n // 4
    x, y = r
    if name == "pow":
        x[:q] = rng.uniform(0, 10, q); y[:q] = rng.uniform(-8, 8, q)
    else:
        x[:q] = rng.uniform(-12, 12, q); y[:q] = rng.uniform(-12, 12, q)
        x[q:q + 1000] = y[q:q + 1000]
    d = _golden()
    if name in BINARY:
        return np.concatenate([d["bx"], x]), np.concatenate([d["by"], y])
    return np.concatenate([d["x"], x]), None


@pytest.mark.parametrize("name", list(TRACED))
def test_traced_program_equals_restatement(oracle, name):
    """The program that the generic body records on this backend (the dry run stored in math_traced.json, recorded over
    mapped CUDAArray<float> arrays by tests/golden/ref_math_traced.cpp) runs on the numpy interpreter for about 4.2
    million arguments and must give the restatement's raw bits wherever the result is not NaN, and NaN where it is."""
    t = _traced()[name]
    (sweep,) = t["program"]["sweeps"]
    assert len(sweep["body"]) == TRACED[name]
    x, y = _inputs(1 << 22, 71 + list(TRACED).index(name), name)
    prog = dict(t["program"], sweeps=[dict(sweep, n=len(x))])
    inputs = {t["x"]: x}
    if y is not None:
        inputs[t["y"]] = y
    emu = Emulator(oracle, inputs)
    emu.run(prog)
    outs = ["frexp_m", "frexp_e"] if name == "frexp" else [name]
    for var, fn in zip(t["out"], outs):
        got = emu.vars[var]
        want = ms.call(fn, x, y) if y is not None else ms.call(fn, x)
        # NaNs are compared as NaNs: which payload survives (and whether a signaling one is quieted) follows the
        # instructions numpy and the C compiler picked, not the recorded program; the device's NaNs are canonical
        bad = ~ms.same_bits(got, want)
        assert not bad.any(), (fn, int(bad.sum()), x[bad][:5], _bits(got)[bad][:5], _bits(want)[bad][:5])


# ------------------------------------------------------------------ recording, lowering, instantiation
def _names(prog, instrs, fast=False):
    return [(prog["fops"] if fast else prog["ops"])[t[0]] for t in instrs]


def _arith(names):
    return [n for n in names if n not in ("NOP", "ST_32", "LOAD_32", "LOAD", "LOADU", "LD_F16", "ST_F16", "LD_U16")]


def _one_sweep(ek):
    prog = ek.debug_program()
    (sw,) = prog["sweeps"]
    assert sw["config"]["fast"] == 1
    return prog, sw


@pytest.mark.parametrize("name", BINARY + UNARY)
def test_each_function_is_one_node_and_one_instruction(ek, name):
    table = {}
    F = _Factory(ek.Float32, table, 0x7f0000000000)
    x, y = F.copy(np.ones(1 << 20, np.float32)), F.copy(np.full(1 << 20, 2, np.float32))
    r = _call(ek, name, x, y) if name in BINARY else _call(ek, name, x)
    want = [name.upper() + "_F32"]
    plan = ek.debug_plan()
    assert plan.count("\n  body ") == 1 and plan.count("sweep ") == 1, plan
    prog, sw = _one_sweep(ek)
    assert _arith(_names(prog, sw["body"])) == want
    assert _arith(_names(prog, sw["fast"]["body"], fast=True)) == want
    assert sw["fast"]["ext"] == MATH_EXT, "the launcher would not pick the instantiation of the new set"
    del r


def test_frexp_is_two_instructions_in_one_sweep(ek):
    table = {}
    x = _Factory(ek.Float32, table, 0x7f0000000000).copy(np.ones(1 << 20, np.float32))
    m, e = ek.frexp(x)
    prog, sw = _one_sweep(ek)
    assert _arith(_names(prog, sw["body"])) == ["FREXP_M_F32", "FREXP_E_F32"]
    assert sw["fast"]["ext"] == MATH_EXT
    del m, e


@pytest.mark.parametrize("name", BINARY)
@pytest.mark.parametrize("form", ["literal_second", "literal_first", "scalar_second", "scalar_first", "array_first"])
def test_uniform_and_reversed_forms(ek, name, form):
    """the second operand a literal or a size-1 (scalar) array: the _UB twin reads one uniform-pool word; the first
    operand one of them while the accumulator holds the second (computed just before): the reversed form's _UB twin; an array
    first operand while the accumulator holds the second: the reversed form"""
    table = {}
    F = _Factory(ek.Float32, table, 0x7f0000000000)
    x, y = F.copy(np.full(1 << 20, 3, np.float32)), F.copy(np.full(1 << 20, 2, np.float32))
    s = F.copy(np.array([0.3], np.float32))
    t = x * 1.5                                               # the accumulator holds t
    u = {"literal_second": lambda: _call(ek, name, t, 2.2), "literal_first": lambda: _call(ek, name, 2.2, t),
         "scalar_second": lambda: _call(ek, name, t, s), "scalar_first": lambda: _call(ek, name, s, t),
         "array_first": lambda: _call(ek, name, y, t)}[form]()
    prog, sw = _one_sweep(ek)
    fast = _arith(_names(prog, sw["fast"]["body"], fast=True))
    op = name.upper() + ("R" if form.endswith("first") else "") + "_F32" + ("" if form == "array_first" else "_UB")
    assert fast == ["MUL_F32_U", op], fast
    assert sw["fast"]["ext"] == MATH_EXT
    del u


@pytest.mark.parametrize("mix,ext", [("pow", 16), ("hypot+erf", 24), ("erfi+tan", 18), ("erf+tanh", 12), ("f16+dawson", 17),
                                     ("pow+f16+tanh+erf+atan2", 31)])
def test_the_launcher_picks_the_smallest_instantiation(ek, mix, ext):
    """ek_fast_ext, the operation sets of the lowered body: the new set alone is EK_FX_MATH (16, run by
    <T, EK_FX_MATH>); mixed with any other set it is run by <T, EK_FX_ALL> (31); a body without it keeps the
    instantiation it ran before (12 and 15: <T, 15>)."""
    table = {}
    x = _Factory(ek.Float32, table, 0x7f0000000000).copy(np.ones(1 << 16, np.float32))
    if "f16" in mix:
        H = _Factory(ek.Float16, table, 0x7c0000000000)
        x = ek.Float32(H.copy(np.ones(1 << 16, np.float16)))
    terms = {"pow": lambda: ek.pow_(x, x * 2.0), "hypot": lambda: ek.hypot(x, x + 1.0), "erf": lambda: ek.erf(x),
             "erfi": lambda: ek.erfi(x), "tan": lambda: ek.tan(x), "tanh": lambda: ek.tanh(x),
             "dawson": lambda: ek.dawson(x), "atan2": lambda: ek.atan2(x, 2.0)}
    r = None
    for k in mix.split("+"):
        if k != "f16":
            r = terms[k]() if r is None else r + terms[k]()
    if "f16" in mix:
        r = ek.Float16(r)
    prog, sw = _one_sweep(ek)
    assert sw["fast"]["ext"] == ext, (mix, sw["fast"]["ext"])
    if "f16" in mix:
        names = _names(prog, sw["fast"]["body"], fast=True)
        assert "LD_F16" in names and "ST_F16" in names, names
    del r


def test_float16_storage_bodies(ek):
    """a Float16 input converted, pow / hypot / frexp computed in Float32, a Float16 output: FOP_LD_F16 and FOP_ST_F16
    around the new operations, one sweep on <T, EK_FX_F16 | EK_FX_MATH>"""
    table = {}
    H = _Factory(ek.Float16, table, 0x7c0000000000)
    a, b = (ek.Float32(H.copy(np.ones(1 << 18, np.float16))) for _ in range(2))
    r = ek.Float16(ek.hypot(ek.pow_(a, 1.5), b) + ek.frexp(a)[0])
    prog, sw = _one_sweep(ek)
    names = _names(prog, sw["fast"]["body"], fast=True)
    assert names.count("LD_F16") == 2 and names.count("ST_F16") == 1, names
    assert {"POW_F32_UB", "FREXP_M_F32"} <= set(names) and ({"HYPOT_F32", "HYPOTR_F32"} & set(names)), names
    assert sw["fast"]["ext"] == MATH_EXT | 1
    del r


@pytest.mark.parametrize("name", BINARY + ("frexp", "dawson", "erfi"))
@pytest.mark.parametrize("cls,tname", [("Float64", "f64"), ("Int32", "i32"), ("UInt32", "u32")])
def test_other_types_are_refused(ek, name, cls, tname):
    table = {}
    F = _Factory(getattr(ek, cls), table, 0x7b0000000000)
    a = F.copy(np.ones(4096, {"Float64": np.float64, "Int32": np.int32, "UInt32": np.uint32}[cls]))
    r = _call(ek, name, a, a) if name in BINARY else getattr(ek, name)(a)
    op = "frexp_m" if name == "frexp" else name
    with pytest.raises(ek.EnokiError) as e:
        ek.debug_plan()
    assert f"op {op} not supported for type {tname}" in str(e.value), str(e.value)
    del r


@pytest.mark.parametrize("name", BINARY + ("frexp", "dawson", "erfi"))
def test_float16_is_refused(ek, name):
    table = {}
    a = _Factory(ek.Float16, table, 0x7c0000000000).copy(np.ones(4096, np.float16))
    r = _call(ek, name, a, a) if name in BINARY else getattr(ek, name)(a)
    op = "frexp_m" if name == "frexp" else name
    with pytest.raises(ek.EnokiError) as e:
        ek.debug_plan()
    assert f"op {op} is not supported on Float16" in str(e.value), str(e.value)
    del r


def test_opcodes_are_appended(ek):
    """after the special functions, which keep their numbers after CBRT"""
    assert [ek.OP[n] for n in ("ERF", "ERFC", "ERFINV", "LGAMMA", "TGAMMA")] == list(range(ek.OP["CBRT"] + 1, ek.OP["CBRT"] + 6))
    new = ["POW", "FREXP_M", "FREXP_E", "HYPOT", "DAWSON", "ERFI"]
    assert [ek.OP_MATH[n] for n in new] == list(range(ek.OP["TGAMMA"] + 1, ek.OP["TGAMMA"] + 7))
    assert ek._OPS_MATH == new and len(ek.OP) == ek.OP["TGAMMA"] + 1 and len(ek.OP_MATH) == len(new)


# ------------------------------------------------------------------ random DAGs: interpreter and host-compiled kernel
_SPECIAL = np.array([0.0, -0.0, 1.0, -1.0, 2.0, 0.5, -3.0, 1e10, np.inf, -np.inf, np.nan, 1e-45, 130.0], np.float32)


def _dag(ek, rng, n, table):
    """A random Float32 DAG mixing the new functions (with literal operands in either position) and erf / tanh / atan2
    from the other sets with add / mul / select; returns [(array, expected numpy value)]"""
    F = _Factory(ek.Float32, table, 0x7f0000000000)
    vals = []
    for _ in range(3):
        x = rng.uniform(-4, 4, n).astype(np.float32)
        x[rng.integers(0, n, max(n // 50, 1))] = rng.choice(_SPECIAL)
        vals.append((F.copy(x), x))
    f = np.float32
    with np.errstate(all="ignore"):
        for _ in range(int(rng.integers(6, 16))):
            k = int(rng.integers(0, 13))
            (a, av), (b, bv) = (vals[int(i)] for i in rng.integers(0, len(vals), 2))
            av, bv = np.broadcast_to(av, (n,)), np.broadcast_to(bv, (n,))
            if k < 4:
                nm = BINARY[k % 2]
                vals.append((_call(ek, nm, a, b), ms.binary(nm, av, bv)))
            elif k == 4:
                c = f(rng.choice([2.2, -1.5, 0.0, 3.0]))
                nm = BINARY[int(rng.integers(0, 2))]
                if rng.integers(0, 2):
                    vals.append((_call(ek, nm, a, float(c)), ms.binary(nm, av, c)))
                else:
                    vals.append((_call(ek, nm, float(c), a), ms.binary(nm, c, av)))
            elif k < 9:
                nm = UNARY[k - 5]
                vals.append((_call(ek, nm, a), ms.unary(nm, av)))
            elif k == 9:
                vals.append((ek.erf(a), ms.ss.unary("erf", av)))
            elif k == 10:
                vals.append((ek.atan2(a, b), ms.ts.atan2(av, bv)))
            elif k == 11:
                vals.append((a * b, (av * bv).astype(f)))
            else:
                vals.append((ek.select(a < b, a, b), np.where(av < bv, av, bv)))
    return vals[3:]


def _dag_case(ek, oracle, seed, emulator):
    rng = np.random.default_rng(7700 + seed)
    n = int(rng.choice([1, 31, 4097, 9000]))
    table = {}
    vals = _dag(ek, rng, n, table)
    keep = [vals[int(i)] for i in rng.choice(len(vals), size=min(4, len(vals)), replace=False)]
    red = ek.hsum(keep[0][0])
    del vals
    prog = ek.debug_program()
    emu = emulator(oracle, table, _Factory.addresses)
    emu.run(prog)
    for arr, want in keep:
        got = emu.vars[arr.index]
        ok = ms.same_bits(got, np.broadcast_to(want, got.shape))
        assert ok.all(), (seed, n, got[~ok][:4], np.broadcast_to(want, got.shape)[~ok][:4])
    assert red.index in emu.vars
    return n


@pytest.mark.parametrize("form", ["assembled", "lowered"])
@pytest.mark.parametrize("seed", range(20))
def test_random_math_dags_on_the_interpreter(ek, oracle, seed, form):
    ms.MathEmulator.prefer_fast = form == "lowered"
    try:
        _dag_case(ek, oracle, seed, ms.MathEmulator)
    finally:
        ms.MathEmulator.prefer_fast = False


@pytest.mark.parametrize("seed", range(20))
def test_random_math_dags_on_the_host_compiled_kernel(ek, oracle, seed):
    before = FastKernelEmulator.native_sweeps
    n = _dag_case(ek, oracle, seed, ms.MathKernelEmulator)
    if n > 1000:
        assert FastKernelEmulator.native_sweeps > before, "no sweep ran on the host-compiled fast kernel"


def test_host_kernel_on_the_golden_arguments(ek, oracle):
    """every function on the arguments of math.npz through the host-compiled kernel, against the restatements, raw
    bits away from NaNs"""
    d = _golden()
    for name in BINARY + UNARY:
        table = {}
        F = _Factory(ek.Float32, table, 0x7f0000000000)
        args = (F.copy(d["bx"]), F.copy(d["by"])) if name in BINARY else (F.copy(d["x"]),)
        r = _call(ek, name, *args)
        emu = ms.MathKernelEmulator(oracle, table, _Factory.addresses)
        before = FastKernelEmulator.native_sweeps
        emu.run(ek.debug_program())
        assert FastKernelEmulator.native_sweeps == before + 1
        got = emu.vars[r.index]
        want = ms.call(name, d["bx"], d["by"]) if name in BINARY else ms.call(name, d["x"])
        assert ms.same_bits(got, want).all(), name
        del r, args
        gc.collect()


# ------------------------------------------------------------------ SASS
def _cuobjdump(obj, *flags):
    path = os.path.join(CSRC, obj)
    if shutil.which("cuobjdump") is None or not os.path.exists(path):
        pytest.skip("cuobjdump or " + obj + " not available")
    return subprocess.run(["cuobjdump", *flags, path], capture_output=True, text=True, check=True).stdout


def _functions(obj):
    """{kernel name (the mangled template name, without the namespace of its translation unit): [SASS instructions]}"""
    fns, cur = {}, None
    for l in _cuobjdump(obj, "-sass").splitlines():
        if "Function :" in l:
            m = re.search(r"(ek_(?:sweep|fast)_kernelI\w*)", l)
            cur = fns.setdefault(m.group(1), []) if m else None
        elif cur is not None:
            m = re.match(r"\s+/\*([0-9a-f]{4,5})\*/\s+(.*?);", l)
            if m:
                cur.append(m.group(2).strip())
    return fns


@pytest.mark.parametrize("T", [128, 256])
@pytest.mark.parametrize("ext", [16, 31])
def test_dispatch_frames_have_no_accumulator_copies(T, ext):
    """the check of tests/test_cpu_trig.py on the instantiations that carry the new operations"""
    from test_cpu_trig import _sass_of
    sass = _sass_of("ek_sweep_fast_trig.o", f"14ek_fast_kernelILi{T}ELj{ext}EEEv11EkSweepArgs")
    fetch = [i for i, l in enumerate(sass) if re.match(r"LDC\.64 R\d+, c\[0x0\]\[R\d+\+0x21[08]\]", l)]
    start = next((i for i in fetch if sum(1 for l in sass[i:i + 40] if re.match(r"@P\d LDS\.128", l)) >= 8), None)
    assert start is not None, "hot-loop fetch not found"
    frame = sass[max(start - 4, 0):start + 45]
    moves = [l for l in frame if re.match(r"(IMAD\.MOV\.U32|MOV) R\d+, (RZ, RZ, )?R\d+", l)]
    assert len(moves) <= 2, "ptxas copies the accumulator in the dispatch frame:\n" + "\n".join(frame)


def test_instantiations_carrying_the_new_operations_use_no_stack():
    """ek_fast_kernel<T, 16>, <T, 31> and ek_sweep_kernel<V, INLINE, true>: no local-memory frame, at most 128
    registers"""
    for obj, pat in (("ek_sweep_fast_trig.o", r"ek_fast_kernelILi(128|256)ELj(16|31)E"),
                     ("ek_sweep_trig.o", r"ek_sweep_kernelILi[48]ELb[01]ELb1E")):
        found = 0
        for block in _cuobjdump(obj, "-res-usage").split("Function ")[1:]:
            name = block.split(":")[0]
            if re.search(pat, name):
                found += 1
                m = re.search(r"STACK:(\d+)", block)
                assert m and int(m.group(1)) == 0, (name, block[:300])
                m = re.search(r"REG:(\d+)", block)
                assert m and int(m.group(1)) <= 128, (name, block[:300])
        assert found == 4, (obj, found)


# SHA-256 of the SASS instructions of every kernel that programs without the new operations run, as nvcc 12.9 compiles
# this repository before and after they were added: ek_sweep.o and ek_sweep_fast.o whole, and every instantiation of
# the fast kernel that existed before them (<T, 2>, <T, 3>, <T, 4>, <T, 7>, <T, 8> and <T, 15>)
PARENT_SASS = {
    "ek_sweep.o|ek_sweep_kernelILi4ELb0ELb0EEEv11EkSweepArgs":
        "80cbeb37d0d8ba26bee4e9dd6a3dc99d62370b931a11d1d427d0386f449a9fcd",
    "ek_sweep.o|ek_sweep_kernelILi4ELb1ELb0EEEv11EkSweepArgs":
        "d3c051ccb2de0bc63c0324144d47d559cc3cb10417a5550d38e4dc5452be4ae1",
    "ek_sweep.o|ek_sweep_kernelILi8ELb0ELb0EEEv11EkSweepArgs":
        "bfba0dc326edf08600a0af4273b27292f42db36f8c981eb0c29c3ac19b27d5d2",
    "ek_sweep.o|ek_sweep_kernelILi8ELb1ELb0EEEv11EkSweepArgs":
        "37a172e5a2f28bdb87da265ea93c8d80c9daa5f37c5c2a27ef229c2dca9657a8",
    "ek_sweep_fast.o|ek_fast_kernelILi128ELj0EEEv11EkSweepArgs":
        "8912f4974ba69ca6ee6fc57fc3ccfc7ee4de374bd98d7670a1049283340edc52",
    "ek_sweep_fast.o|ek_fast_kernelILi128ELj1EEEv11EkSweepArgs":
        "f62a4d59315d34b8b9680b6cd6f661daa29651efdc7b348c8b1685561bc4ab3c",
    "ek_sweep_fast.o|ek_fast_kernelILi256ELj0EEEv11EkSweepArgs":
        "264b28e006f01902d4faed165a29fb93e6f396224040a9cfaa5c293d6af86bef",
    "ek_sweep_fast.o|ek_fast_kernelILi256ELj1EEEv11EkSweepArgs":
        "f6f436d777affe2b201fb543ff40da730e4df0059a578ab5a880a6314636a4de",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi128ELj2EEEv11EkSweepArgs":
        "56c20f48ad13b223007f86ebde19d7ee1f650a665de0b573491e69bf353ca089",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi128ELj3EEEv11EkSweepArgs":
        "9d7fc2d05c7221677aead2824718ab02d006430325435df9f631932722c12d66",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi128ELj4EEEv11EkSweepArgs":
        "026da432cafb464d72c397ce5d10f9fd2accd2c2869383bac969b3f9fb3f03cc",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi128ELj7EEEv11EkSweepArgs":
        "6981518b309e3379b9c66b9bd92f607a73840959f17039ee4f62467be9fed16b",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi128ELj8EEEv11EkSweepArgs":
        "7fd1a2ebf4f11742f88e88c0f566fae357f5fc22a83a4e89d60f4812fc799cc5",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi256ELj2EEEv11EkSweepArgs":
        "f4e7cf59785c2582843d9e7f4a874a91bdf5b976b591183d71f8f089a26fff5c",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi256ELj3EEEv11EkSweepArgs":
        "f167adf330ab54a721463ae7e694981d7acdb3da8848a4953e92d86a48a2947d",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi256ELj4EEEv11EkSweepArgs":
        "0f734899cdbc077ab21c152ff1ce5c77d6fff9c31bb7bd2a8553e3c4c4639a4e",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi256ELj7EEEv11EkSweepArgs":
        "d7b0253e8fe26ca093a3836400b0c8974b6486a0c2709cfd760b1e200512cfec",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi256ELj8EEEv11EkSweepArgs":
        "d83fd6e08989c95f99dbc2d88302e2549632e2be5ff23e5851cc6939c4ffe744",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi128ELj15EEEv11EkSweepArgs":
        "0ee6dcbb7ce7c54610046dc4234b1e683efb715df7f2f1dc9eacab53c78f2e67",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi256ELj15EEEv11EkSweepArgs":
        "447cf1d6d122d60dd50686dae67256eb4d60257c404c5bfa9893f90a4068a6f5",
}


def _nvcc_release():
    if shutil.which("nvcc") is None:
        return None
    m = re.search(r"release (\d+\.\d+)", subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout)
    return m and m.group(1)


def _digest(lines):
    return hashlib.sha256("\n".join(lines).encode()).hexdigest()


@pytest.mark.parametrize("obj", ["ek_sweep.o", "ek_sweep_fast.o", "ek_sweep_fast_trig.o"])
def test_kernels_of_other_programs_are_unchanged(obj):
    """Adding cases to a kernel that other programs run costs them time (1.5-3 % on an H100 when the hyperbolic cases
    were added to the trigonometric instantiations); these kernels compile to the same instructions as before the new
    operations existed."""
    if _nvcc_release() != "12.9":
        pytest.skip("the digests are of nvcc 12.9's SASS")
    want = {k.split("|")[1]: v for k, v in PARENT_SASS.items() if k.split("|")[0] == obj}
    fns = _functions(obj)
    assert want and set(want) <= set(fns)
    for name, digest in want.items():
        assert _digest(fns[name]) == digest, name
