"""CPU: the Float32 trigonometric operations tan, cot, asin, acos, atan and atan2 (EK_OP_TAN ... EK_OP_ATAN2).
What the planner records and lowers for them (ek_debug_program), the operations it refuses, the C restatements of
tests/trig_oracle.c against the reference CPU path (tests/golden/unary.npz, tests/golden/trig.npz), and random expression
DAGs that contain them on the numpy interpreter and on the host-compiled fast kernel (tests/cpu_kernel), bit for bit."""
import gc
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

import trig_support as ts
from fast_kernel_emu import FastKernelEmulator
from test_cpu_emulator import _Factory

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
DOP = {"tan": "TAN_F32", "cot": "COT_F32", "asin": "ASIN_F32", "acos": "ACOS_F32", "atan": "ATAN_F32"}


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


def _ulps(a, b):
    ai = _bits(a).view(np.int32).astype(np.int64); bi = _bits(b).view(np.int32).astype(np.int64)
    ai = np.where(ai < 0, -(ai & 0x7fffffff), ai); bi = np.where(bi < 0, -(bi & 0x7fffffff), bi)
    return np.abs(ai - bi)


# ------------------------------------------------------------------ the C restatements against the reference CPU path
def _check_against_reference(name, x, ref):
    got = ts.unary(name, x)
    if name in ("tan", "cot"):
        # the reference computes rcp with rcpps + one Newton step (array_avx.h), the backend and the restatement with the
        # correctly rounded quotient: exact where no reciprocal is taken, within that bound where it is
        alt, recip = ts.tancot_rcp(name, x, 1)
        assert (_bits(alt) == _bits(got)).all(), "the float quotient is not the correctly rounded reciprocal"
        plain = ~recip
        assert (_bits(got)[plain] == _bits(ref)[plain]).all(), (name, x[plain][_bits(got)[plain] != _bits(ref)[plain]][:5])
        finite = recip & np.isfinite(ref) & np.isfinite(got)
        assert (_ulps(got[finite], ref[finite]) <= 2).all(), (name, int(_ulps(got[finite], ref[finite]).max()))
        # rcpps returns inf for zero and denormal arguments, and its Newton step then gives NaN (0 * inf): only results
        # of at least 2^126 in magnitude, the reciprocals of such arguments, may differ in kind
        tiny = recip & ~(np.abs(got) < np.float32(2.0 ** 126))
        assert (np.isnan(got) == np.isnan(ref))[recip & ~tiny].all()
        assert (np.isinf(got) == np.isinf(ref))[recip & ~tiny].all()
    else:
        bad = _bits(got) != _bits(ref)
        assert not bad.any(), (name, x[bad][:5], got[bad][:5], ref[bad][:5])


@pytest.mark.parametrize("name", ["tan", "asin", "acos", "atan"])
def test_restatement_against_unary_golden(name):
    d = np.load(os.path.join(GOLDEN, "unary.npz"))
    _check_against_reference(name, d["x"], d[name])


@pytest.mark.parametrize("name", ["tan", "cot", "asin", "acos", "atan"])
def test_restatement_against_trig_golden(name):
    d = np.load(os.path.join(GOLDEN, "trig.npz"))
    _check_against_reference(name, d["x"], d[name])


def test_atan2_restatement_against_trig_golden():
    d = np.load(os.path.join(GOLDEN, "trig.npz"))
    y, x, ref = d["y2"], d["x2"], d["atan2"]
    got = ts.atan2(y, x)
    nan_in = np.isnan(y) | np.isnan(x)
    bad = (_bits(got) != _bits(ref)) & ~nan_in
    assert not bad.any(), (y[bad][:5], x[bad][:5], got[bad][:5], ref[bad][:5])
    # a NaN operand: the evaluator's min / max return their second operand when one is NaN, array_avx.h's min_ / max_
    # their first (DESIGN.md §4), so where the other operand is 0 the selected max(|x|, |y|) is 0 here and the result +0
    assert (np.isnan(got) | ((got == 0) & (np.minimum(np.abs(np.nan_to_num(y)), np.abs(np.nan_to_num(x))) == 0)))[nan_in].all()


def test_atan_is_atan2_with_one():
    x = np.random.default_rng(3).integers(0, 1 << 32, 100_000, dtype=np.uint64).astype(np.uint32).view(np.float32)
    assert (_bits(ts.unary("atan", x)) == _bits(ts.atan2(x, np.float32(1)))).all()


# ------------------------------------------------------------------ recording, lowering, instantiation
def _names(prog, instrs, fast=False):
    return [(prog["fops"] if fast else prog["ops"])[t[0]] for t in instrs]


def _arith(names):
    return [n for n in names if n not in ("NOP", "ST_32", "LOAD_32", "LOAD", "LOADU", "LD_F16", "ST_F16", "LD_U16")]


@pytest.mark.parametrize("name", ["tan", "cot", "asin", "acos", "atan", "atan2"])
def test_each_function_is_one_node_and_one_instruction(ek, name):
    table = {}
    F = _Factory(ek.Float32, table, 0x7f0000000000)
    a, b = F.copy(np.ones(8192, np.float32)), F.copy(np.ones(8192, np.float32))
    r = ek.atan2(a, b) if name == "atan2" else getattr(ek, name)(a)
    plan = ek.debug_plan()
    assert plan.count("\n  body ") >= 1
    prog = ek.debug_program()
    (sw,) = prog["sweeps"]
    want = "ATAN2_F32" if name == "atan2" else DOP[name]
    assert _arith(_names(prog, sw["body"])) == [want], _names(prog, sw["body"])
    assert sw["config"]["fast"] == 1
    assert _arith(_names(prog, sw["fast"]["body"], fast=True)) == [want]
    assert sw["fast"]["ext"] == 2, "the launcher would not pick the trigonometric instantiation"
    del r


@pytest.mark.parametrize("which", ["y", "x"])
@pytest.mark.parametrize("kind", ["literal", "scalar"])
def test_atan2_with_a_uniform_operand_uses_the_uniform_twin(ek, which, kind):
    table = {}
    F = _Factory(ek.Float32, table, 0x7f0000000000)
    a = F.copy(np.linspace(-3, 3, 8192).astype(np.float32))
    u = ek.Float32(0.75) if kind == "literal" else F.copy(np.array([0.75], np.float32))
    r = ek.atan2(u, a) if which == "y" else ek.atan2(a, u)
    prog = ek.debug_program()
    sw = [s for s in prog["sweeps"] if s["n"] == 8192][0]
    fast = _names(prog, sw["fast"]["body"], fast=True)
    trig = _arith(fast)
    assert len(trig) == 1 and trig[0].startswith("ATAN2"), fast
    # the uniform operand is one pool word: the _U twin's operand, or the accumulator loaded by LOADU
    assert trig[0].endswith("_U") or "LOADU" in fast, fast
    del r


def _c2(ek, F):
    x0, x1, x2, x3 = (F.copy(np.ones(1 << 16, np.float32)) for _ in range(4))
    t = ek.fmadd(x0, x1, x2)
    return ek.fmadd(ek.sin(ek.fmadd(x3, ek.exp(-(t * t)), x0)), x1, ek.sqrt(abs(t)))


def test_float32_c2_keeps_the_base_instantiation(ek):
    table = {}
    r = _c2(ek, _Factory(ek.Float32, table, 0x7f0000000000))
    (sw,) = ek.debug_program()["sweeps"]
    assert sw["config"]["fast"] == 1 and sw["fast"]["ext"] == 0
    del r


def test_float16_storage_with_atan2_needs_both_sets(ek):
    table = {}
    H = _Factory(ek.Float16, table, 0x7c0000000000)
    y, x = (ek.Float32(H.copy(np.ones(1 << 16, np.float16))) for _ in range(2))
    r = ek.Float16(ek.atan2(y, x))
    prog = ek.debug_program()
    (sw,) = prog["sweeps"]
    fast = _names(prog, sw["fast"]["body"], fast=True)
    assert fast.count("LD_F16") == 2 and fast[-1] == "ST_F16" and any(f.startswith("ATAN2") for f in fast), fast
    assert sw["config"]["fast"] == 1 and sw["fast"]["ext"] == 3
    del r


@pytest.mark.parametrize("name", ["tan", "cot", "asin", "acos", "atan", "atan2"])
@pytest.mark.parametrize("cls,tname", [("Float64", "f64"), ("Int32", "i32")])
def test_other_types_are_refused(ek, name, cls, tname):
    table = {}
    C = getattr(ek, cls)
    F = _Factory(C, table, 0x7b0000000000)
    dt = np.float64 if cls == "Float64" else np.int32
    a, b = F.copy(np.ones(4096, dt)), F.copy(np.ones(4096, dt))
    r = ek.atan2(a, b) if name == "atan2" else getattr(ek, name)(a)
    with pytest.raises(ek.EnokiError) as e:
        ek.debug_plan()
    assert f"op {name} not supported for type {tname}" in str(e.value), str(e.value)
    del r


# ------------------------------------------------------------------ random DAGs: interpreter and host-compiled kernel
def _dag(ek, rng, n, table):
    """A random Float32 DAG mixing the six functions (atan2 with array, literal and scalar operands in both positions)
    with add / sub / mul / select; returns [(array, expected numpy value)]"""
    F = _Factory(ek.Float32, table, 0x7f0000000000)
    vals = []
    for _ in range(3):
        x = rng.uniform(-3, 3, n).astype(np.float32)
        x[rng.integers(0, n, max(n // 50, 1))] = rng.choice(np.array([0.0, -0.0, 1.0, -1.0, 0.5, np.inf, -np.inf, np.nan, 1e-30], np.float32))
        vals.append((F.copy(x), x))
    s = np.float32(rng.uniform(-2, 2))
    scalar = (F.copy(np.array([s], np.float32)), s)
    with np.errstate(all="ignore"):
        for _ in range(int(rng.integers(6, 16))):
            k = int(rng.integers(0, 10))
            (a, av), (b, bv) = (vals[int(i)] for i in rng.integers(0, len(vals), 2))
            if k < 5:
                name = ("tan", "cot", "asin", "acos", "atan")[k]
                vals.append((getattr(ek, name)(a), ts.unary(name, np.broadcast_to(av, (n,)))))
            elif k == 5:
                vals.append((ek.atan2(a, b), ts.atan2(av, bv)))
            elif k == 6:
                lit = np.float32(rng.choice([0.5, -2.0, 0.0, 3.0]))
                u, uv = (ek.Float32(float(lit)), lit) if rng.integers(0, 2) else scalar
                if rng.integers(0, 2):
                    vals.append((ek.atan2(u, a), ts.atan2(np.broadcast_to(uv, (n,)), av)))
                else:
                    vals.append((ek.atan2(a, u), ts.atan2(av, np.broadcast_to(uv, (n,)))))
            elif k == 7:
                vals.append((a * b, (av * bv).astype(np.float32)))
            elif k == 8:
                vals.append((a - b, (av - bv).astype(np.float32)))
            else:
                vals.append((ek.select(a < b, a, b + 1.0), np.where(av < bv, av, (bv + np.float32(1)).astype(np.float32))))
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
        want = np.broadcast_to(want, got.shape)
        ok = ts.same_bits(got, want)
        assert ok.all(), (seed, n, got[~ok][:4], want[~ok][:4])
    assert red.index in emu.vars
    return n


@pytest.mark.parametrize("form", ["assembled", "lowered"])
@pytest.mark.parametrize("seed", range(40))
def test_random_trig_dags_on_the_interpreter(ek, oracle, seed, form):
    ts.TrigEmulator.prefer_fast = form == "lowered"
    try:
        _dag_case(ek, oracle, seed, ts.TrigEmulator)
    finally:
        ts.TrigEmulator.prefer_fast = False


@pytest.mark.parametrize("seed", range(40))
def test_random_trig_dags_on_the_host_compiled_kernel(ek, oracle, seed):
    before = FastKernelEmulator.native_sweeps
    n = _dag_case(ek, oracle, seed, ts.TrigKernelEmulator)
    if n > 1000:
        assert FastKernelEmulator.native_sweeps > before, "no sweep ran on the host-compiled fast kernel"


def test_random_trig_dags_on_the_128_thread_kernel():
    """The host-compiled kernel once more restricted to T = 128 (EK_FAST_T is read once per process: a child process)."""
    env = dict(os.environ, EK_FAST_T="128")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_cpu_trig.py"), "-q", "-x",
                        "-k", "host_compiled_kernel", "-p", "no:cacheprovider"], capture_output=True, text=True,
                       timeout=1800, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout


def test_host_kernel_on_every_special_and_branch_value(ek, oracle):
    """tan / cot / asin / acos / atan on the branch-point values of trig.npz and atan2 on its special cross product,
    through the host-compiled kernel, against the restatements"""
    d = np.load(os.path.join(GOLDEN, "trig.npz"))
    for name in ("tan", "cot", "asin", "acos", "atan", "atan2"):
        table = {}
        F = _Factory(ek.Float32, table, 0x7f0000000000)
        if name == "atan2":
            y, x = d["y2"], d["x2"]
            r = ek.atan2(F.copy(y), F.copy(x)); want = ts.atan2(y, x)
        else:
            x = d["x"]
            r = getattr(ek, name)(F.copy(x)); want = ts.unary(name, x)
        prog = ek.debug_program()
        emu = ts.TrigKernelEmulator(oracle, table, _Factory.addresses)
        emu.run(prog)
        got = emu.vars[r.index]
        assert (_bits(got) == _bits(want)).all(), name
        del r
        gc.collect()


# ------------------------------------------------------------------ SASS
CSRC = os.path.join(ROOT, "enoki_b200", "csrc")


def _sass_of(obj, suffix):
    obj = os.path.join(CSRC, obj)
    if shutil.which("cuobjdump") is None or not os.path.exists(obj):
        pytest.skip("cuobjdump or " + os.path.basename(obj) + " not available")
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    on, lines = False, []
    for l in out.splitlines():
        if "Function :" in l:
            on = l.strip().endswith(suffix)
        elif on:
            m = re.match(r"\s+/\*([0-9a-f]{4,5})\*/\s+(.*?);", l)
            if m:
                lines.append(m.group(2).strip())
    assert lines, suffix + " not found in the object"
    return lines


@pytest.mark.parametrize("T", [128, 256])
@pytest.mark.parametrize("ext", [0, 1, 2, 3])
def test_dispatch_frames_have_no_accumulator_copies(T, ext):
    # (the trigonometric instantiations are compiled into a module of their own, ek_sweep_fast_trig.o)
    sass = _sass_of("ek_sweep_fast_trig.o" if ext & 2 else "ek_sweep_fast.o", f"14ek_fast_kernelILi{T}ELj{ext}EEEv11EkSweepArgs")
    fetch = [i for i, l in enumerate(sass) if re.match(r"LDC\.64 R\d+, c\[0x0\]\[R\d+\+0x21[08]\]", l)]
    start = next((i for i in fetch if sum(1 for l in sass[i:i + 40] if re.match(r"@P\d LDS\.128", l)) >= 8), None)
    assert start is not None, "hot-loop fetch not found"
    frame = sass[max(start - 4, 0):start + 45]
    moves = [l for l in frame if re.match(r"(IMAD\.MOV\.U32|MOV) R\d+, (RZ, RZ, )?R\d+", l)]
    assert len(moves) <= 2, "ptxas copies the accumulator in the dispatch frame:\n" + "\n".join(frame)


@pytest.mark.parametrize("obj,kernel,n", [("ek_sweep_fast.o", "ek_fast_kernel", 4), ("ek_sweep.o", "ek_sweep_kernel", 4)])
def test_base_modules_hold_only_the_kernels_without_trig(obj, kernel, n):
    """the modules every other program runs from keep exactly the kernels they had before the trigonometric operations:
    those are instantiated in ek_sweep_fast_trig.o / ek_sweep_trig.o"""
    path = os.path.join(CSRC, obj)
    if shutil.which("cuobjdump") is None or not os.path.exists(path):
        pytest.skip("cuobjdump or " + obj + " not available")
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    names = [l.split("Function :")[1].strip() for l in out.splitlines() if "Function :" in l and kernel in l]
    assert len(names) == n, names
    if kernel == "ek_fast_kernel":        # <T, 0> and <T, EK_FX_F16> only
        assert all(re.search(r"ILi(128|256)ELj[01]EEEv", s) for s in names), names
    else:                                 # <V, INLINE, false> only
        assert all(re.search(r"ILi[48]ELb[01]ELb0EEEv", s) for s in names), names
