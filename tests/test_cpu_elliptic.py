"""CPU: the Float32 Carlson integrals carlson_rf, carlson_rd and carlson_rc (EK_OP_CARLSON_RF ... EK_OP_CARLSON_RC).
What the planner records and lowers for them (ek_debug_program): one instruction each, x loaded by the instruction when
the accumulator holds y or z, the reversed carlson_rc, uniform operands, the instantiation the launcher picks; the
operations it refuses; the C restatements of tests/ell_oracle.c against one loop pass and the epilogue recorded on this
backend one primitive per operation (tests/golden/ell_traced.json, run on the numpy interpreter with the loop driven
from here) and against SciPy; random
expression DAGs that contain them on the host-compiled fast kernel (tests/cpu_kernel), bit for bit; and the SASS of the
kernels that carry them and of those that must not change."""
import gc
import json
import os
import re

import numpy as np
import pytest

import ell_support as es
import math_support as ms
from ek_emulator import Emulator
from fast_kernel_emu import FastKernelEmulator
from test_cpu_emulator import _Factory
from test_cpu_math import PARENT_SASS, _cuobjdump, _digest, _functions, _nvcc_release

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
NAMES = es.TERNARY + es.BINARY
ELL_EXT = 32


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
    return np.load(os.path.join(GOLDEN, "ell.npz"))


def _traced():
    with open(os.path.join(GOLDEN, "ell_traced.json")) as f:
        return json.load(f)


def _names(prog, instrs, fast=False):
    return [(prog["fops"] if fast else prog["ops"])[t[0]] for t in instrs]


def _arith(names):
    return [n for n in names if n not in ("NOP", "ST_32", "LOAD_32", "LOAD", "LOADU", "LD_F16", "ST_F16", "LD_U16")]


def _one_sweep(ek):
    prog = ek.debug_program()
    (sw,) = prog["sweeps"]
    assert sw["config"]["fast"] == 1
    return prog, sw


def _arrays(ek, arity, n=1 << 20):
    F = _Factory(ek.Float32, {}, 0x7f0000000000)
    return [F.copy(np.full(n, 1 + k, np.float32)) for k in range(arity)]


# ------------------------------------------------------------------ recording, lowering, instantiation
def test_opcodes_are_appended(ek):
    """after the math set, which keeps its numbers after TGAMMA; OP and OP_MATH are as they were"""
    new = ["CARLSON_RF", "CARLSON_RD", "CARLSON_RC"]
    assert [ek.OP_ELL[n] for n in new] == list(range(ek.OP_MATH["ERFI"] + 1, ek.OP_MATH["ERFI"] + 4))
    assert ek._OPS_ELL == new and len(ek.OP_ELL) == 3
    assert len(ek.OP) == ek.OP["TGAMMA"] + 1 and len(ek.OP_MATH) == 6


@pytest.mark.parametrize("name", NAMES)
def test_each_function_is_one_instruction(ek, name):
    args = _arrays(ek, 3 if name in es.TERNARY else 2)
    r = getattr(ek, name)(*args)
    plan = ek.debug_plan()
    assert plan.count("\n  body ") == 1 and plan.count("sweep ") == 1, plan
    prog, sw = _one_sweep(ek)
    want = [name.upper() + "_F32"]
    assert _arith(_names(prog, sw["body"])) == want
    assert _arith(_names(prog, sw["fast"]["body"], fast=True)) == want
    assert sw["fast"]["ext"] == ELL_EXT, "the launcher would not pick the instantiation of the new set"
    del r


def test_comp_ellint_1_is_one_sweep_with_uniform_x_and_z(ek):
    """comp_ellint_1(k) = carlson_rf(0, 1 - k^2, 1): k * k, 1 - k^2, then the integral with the literals 0 and 1
    broadcast from the uniform pool (FF_BU / FF_CU) -- one sweep, three body instructions"""
    (k,) = _arrays(ek, 1)
    r = ek.comp_ellint_1(k)
    prog, sw = _one_sweep(ek)
    assert _arith(_names(prog, sw["body"])) == ["MUL_F32", "SUBR_F32", "CARLSON_RF_F32"]
    fast = sw["fast"]["body"]
    names = _names(prog, fast, fast=True)
    i = names.index("CARLSON_RF_F32")
    assert names[i - 1] == "LOADU", names                # x = 0: a uniform accumulator load
    flags = fast[i][1]
    assert flags & 0x8 and flags & 0x1, hex(flags)       # FF_CU: z = 1 from the pool, FF_B: y from a slot
    assert sw["fast"]["ext"] == ELL_EXT
    del r


@pytest.mark.parametrize("name", es.TERNARY)
def test_x_is_loaded_when_the_accumulator_holds_y_or_z(ek, name):
    x, y, z = _arrays(ek, 3)
    for make in (lambda: (x, y * 2.0, z), lambda: (x, y, z * 2.0)):
        r = getattr(ek, name)(*make())
        prog, sw = _one_sweep(ek)
        body = sw["body"]
        names = _names(prog, body)
        assert _arith(names) == ["MUL_F32", name.upper() + "_F32"], names
        ins = body[names.index(name.upper() + "_F32")]
        assert ins[1] & 0x80, "x is not loaded by the instruction (EKF_HAS_A)"
        del r
        gc.collect()
        ek.lib().ek_debug_discard_side_effects()


@pytest.mark.parametrize("form", ["array", "reversed", "literal_x", "literal_y"])
def test_carlson_rc_forms(ek, form):
    x, y = _arrays(ek, 2)
    r = {"array": lambda: ek.carlson_rc(x, y), "reversed": lambda: ek.carlson_rc(x, y * 2.0),
         "literal_x": lambda: ek.carlson_rc(0.5, y), "literal_y": lambda: ek.carlson_rc(x, 2.0)}[form]()
    prog, sw = _one_sweep(ek)
    fast = _arith(_names(prog, sw["fast"]["body"], fast=True))
    op = "CARLSON_RCR_F32" if form == "reversed" else "CARLSON_RC_F32"
    assert fast[-1] == op, fast
    assert sw["fast"]["ext"] == ELL_EXT
    del r


@pytest.mark.parametrize("mix,ext", [("rf", 32), ("rc+erf", 40), ("rd+hypot", 48), ("rc+atan2+f16", 35),
                                     ("pow+f16+tanh+erf+atan2", 31), ("hypot+erf", 24), ("rf+pow+f16+tanh+erf+atan2", 63)])
def test_the_launcher_picks_the_smallest_instantiation(ek, mix, ext):
    """ek_fast_ext: the Carlson set alone is EK_FX_ELL (32, <T, 32>); mixed with any other set <T, 63>; a body without
    it keeps the instantiation and ext it had (31, 24)"""
    table = {}
    x = _Factory(ek.Float32, table, 0x7f0000000000).copy(np.ones(1 << 16, np.float32))
    if "f16" in mix:
        x = ek.Float32(_Factory(ek.Float16, table, 0x7c0000000000).copy(np.ones(1 << 16, np.float16)))
    terms = {"rf": lambda: ek.carlson_rf(x, x * 2.0, 3.0), "rd": lambda: ek.carlson_rd(x, 1.0, x + 1.0),
             "rc": lambda: ek.carlson_rc(x, 2.0), "erf": lambda: ek.erf(x), "hypot": lambda: ek.hypot(x, x + 1.0),
             "atan2": lambda: ek.atan2(x, 2.0), "pow": lambda: ek.pow_(x, x * 2.0), "tanh": lambda: ek.tanh(x)}
    r = None
    for k in mix.split("+"):
        if k != "f16":
            r = terms[k]() if r is None else r + terms[k]()
    if "f16" in mix:
        r = ek.Float16(r)
    prog, sw = _one_sweep(ek)
    assert sw["fast"]["ext"] == ext, (mix, sw["fast"]["ext"])
    del r


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("cls,tname", [("Float64", "f64"), ("Int32", "i32"), ("UInt32", "u32")])
def test_other_types_are_refused(ek, name, cls, tname):
    F = _Factory(getattr(ek, cls), {}, 0x7b0000000000)
    a = F.copy(np.ones(4096, {"Float64": np.float64, "Int32": np.int32, "UInt32": np.uint32}[cls]))
    r = getattr(ek, name)(*([a] * (3 if name in es.TERNARY else 2)))
    with pytest.raises(ek.EnokiError) as e:
        ek.debug_plan()
    assert f"op {name} not supported for type {tname}" in str(e.value), str(e.value)
    del r


@pytest.mark.parametrize("name", NAMES)
def test_float16_is_refused(ek, name):
    a = _Factory(ek.Float16, {}, 0x7c0000000000).copy(np.ones(4096, np.float16))
    r = getattr(ek, name)(*([a] * (3 if name in es.TERNARY else 2)))
    with pytest.raises(ek.EnokiError) as e:
        ek.debug_plan()
    assert f"op {name} is not supported on Float16" in str(e.value), str(e.value)
    del r


# ------------------------------------------------------------------ the restatements are the traced bodies
def _valid(n, seed, arity):
    rng = np.random.default_rng(seed)
    a = np.exp2(rng.uniform(-40, 40, (arity, n))).astype(np.float32)
    a[0, ::10] = 0
    return list(a)


def _specials(arity):
    s = np.array([0.0, 1e-45, 1e-40, 1.17549435e-38, 1e-30, 1e-4, 0.5, 1.0, 2.0, 1e4, 1e30, 3.4028235e38, np.inf, np.nan],
                 np.float32)
    s = np.concatenate([s, -s[1:]])
    return [g.ravel() for g in np.meshgrid(*([s] * arity), indexing="ij")]


def _run(oracle, prog, inputs):
    emu = Emulator(oracle, inputs)
    emu.run(prog)
    return emu.vars


def _traced_function(oracle, name, args):
    """the duplication loop with the recorded pass and epilogue programs: passes until no element is active or ten
    passes have run, as special.h drives its loop, then the epilogue on the last pass's XYZ and mu_inv (s and inv_mu)"""
    t = _traced()
    key = {"carlson_rf": "rf", "carlson_rd": "rd", "carlson_rc": "rc"}[name]
    p, e = t[key + "_pass"], t[key + "_tail"]
    n = len(args[0])
    sweep = lambda prog: dict(prog, sweeps=[dict(s, n=n) for s in prog["sweeps"]])
    pprog, eprog = sweep(p["program"]), sweep(e["program"])
    state = dict(zip("xyz", args))
    state["active"] = np.ones(n, np.bool_)
    if name == "carlson_rd":
        state["sum"], state["num"] = np.zeros(n, np.float32), np.ones(n, np.float32)
    for it in range(1, 11):
        vars_ = _run(oracle, pprog, {p["in"][r]: state[r] for r in p["in"]})
        out = {r: np.asarray(vars_[v]) for r, v in p["out"].items()}
        if not out["active"].astype(bool).any() or it == 10:
            break
        state.update({r: out[r] for r in state})
        state["active"] = out["active"].astype(np.bool_)
    # (the last pass's XYZ and mu_inv; sum and num as they were before its update, which special.h does not make)
    vars_ = _run(oracle, eprog, {e["in"][r]: (state[r] if r in state else out[r]) for r in e["in"]})
    return np.asarray(vars_[e["out"]["r"]])


@pytest.mark.parametrize("name", NAMES)
def test_traced_program_equals_restatement(oracle, name):
    """The pass and the epilogue recorded one primitive per operation over the backend's own arrays
    (tests/golden/ell_traced.cpp -> ell_traced.json), driven from here, on the numpy interpreter: 2^20 valid arguments
    plus the cross product of special values must give the C restatement's raw bits wherever the result is not NaN, and
    NaN where it is.  That the sequence is the one special.h's templates record is checked on the device against the
    templates themselves (tests/cpp/ell_check.cpp)."""
    arity = 3 if name in es.TERNARY else 2
    v, s = _valid(1 << 20, 17 + NAMES.index(name), arity), _specials(arity)
    args = [np.concatenate([a, b]) for a, b in zip(v, s)]
    with np.errstate(all="ignore"):
        got = _traced_function(oracle, name, args)
    want = es.call(name, *args)
    bad = ~es.same_bits(got, want)
    assert not bad.any(), (name, int(bad.sum()), [a[bad][:5] for a in args], _bits(got)[bad][:5], _bits(want)[bad][:5])


def test_restatement_against_scipy():
    """An independent check of what the restatement (and so the device) computes: SciPy's elliprf / elliprd / elliprc
    and ellipk / ellipe / ellipkinc / ellipeinc (whose parameter is m = k^2) in double precision, on valid arguments over
    2^-40 ... 2^40, within a relative 2e-6 (the duplication loop stops at eps^(1/6) of float, the series is truncated)"""
    sp = pytest.importorskip("scipy.special")
    bound = 2e-6
    x, y, z = _valid(1 << 16, 3, 3)
    for name, ref in (("carlson_rf", sp.elliprf), ("carlson_rd", sp.elliprd)):
        got = es.call(name, x, y, z).astype(np.float64)
        want = ref(x.astype(np.float64), y.astype(np.float64), z.astype(np.float64))
        assert np.max(np.abs(got / want - 1)) < bound, name
    got = es.call("carlson_rc", x, y).astype(np.float64)
    want = sp.elliprc(x.astype(np.float64), y.astype(np.float64))
    assert np.max(np.abs(got / want - 1)) < bound, "carlson_rc"
    rng = np.random.default_rng(4)
    f = np.float32
    k = rng.uniform(-0.999, 0.999, 1 << 14).astype(f)
    phi = rng.uniform(-1.5, 1.5, 1 << 14).astype(f)
    k2 = (k * k).astype(f)
    rf, rd = es.call("carlson_rf", 0, (f(1) - k2).astype(f), 1), es.call("carlson_rd", 0, (f(1) - k2).astype(f), 1)
    m = k.astype(np.float64) ** 2
    assert np.max(np.abs(rf / sp.ellipk(m) - 1)) < bound
    assert np.max(np.abs((rf - (f(1.0 / 3.0) * k2).astype(f) * rd).astype(f) / sp.ellipe(m) - 1)) < bound
    # ellint_1 / ellint_2 for |phi| < pi / 2 (special.h's loop-free branch), sin / cos in double here
    s, c = np.sin(phi.astype(np.float64)).astype(f), np.cos(phi.astype(np.float64)).astype(f)
    xyz = ((c * c).astype(f), (f(1) - (k2 * s).astype(f) * s).astype(f), np.ones_like(s))
    e1 = (s * es.call("carlson_rf", *xyz)).astype(np.float64)
    w1 = sp.ellipkinc(phi.astype(np.float64), m)
    assert np.max(np.abs(e1 - w1) / np.maximum(np.abs(w1), 1e-3)) < 1e-5
    sk = ((s * s).astype(f) * k2).astype(f)
    xyz = ((c * c).astype(f), (f(1) - sk).astype(f), np.ones_like(s))
    e2 = (s * (es.call("carlson_rf", *xyz) - (f(1.0 / 3.0) * sk).astype(f) * es.call("carlson_rd", *xyz))).astype(np.float64)
    w2 = sp.ellipeinc(phi.astype(np.float64), m)
    assert np.max(np.abs(e2 - w2) / np.maximum(np.abs(w2), 1e-3)) < 1e-5


# ------------------------------------------------------------------ random DAGs on the host-compiled kernel
_SPECIAL = np.array([0.0, 1.0, 2.0, 0.5, 1e10, 1e-30, np.inf, np.nan, -1.0], np.float32)


def _dag(ek, rng, n, table):
    """A random Float32 DAG mixing the Carlson integrals (literal operands in any position) with erf, hypot and atan2
    and add / mul / select; returns [(array, expected numpy value)]"""
    F = _Factory(ek.Float32, table, 0x7f0000000000)
    vals = []
    for _ in range(3):
        x = np.exp2(rng.uniform(-8, 8, n)).astype(np.float32)
        x[rng.integers(0, n, max(n // 50, 1))] = rng.choice(_SPECIAL)
        vals.append((F.copy(x), x))
    f = np.float32
    with np.errstate(all="ignore"):
        for _ in range(int(rng.integers(6, 14))):
            k = int(rng.integers(0, 9))
            (a, av), (b, bv), (c, cv) = (vals[int(i)] for i in rng.integers(0, len(vals), 3))
            av, bv, cv = (np.broadcast_to(v, (n,)) for v in (av, bv, cv))
            if k < 2:
                nm = es.TERNARY[k]
                if rng.integers(0, 2):
                    lit = f(rng.choice([0.0, 1.0, 2.5]))
                    vals.append((getattr(ek, nm)(a, float(lit), c), es.call(nm, av, lit, cv)))
                else:
                    vals.append((getattr(ek, nm)(a, b, c), es.call(nm, av, bv, cv)))
            elif k == 2:
                vals.append((ek.carlson_rc(a, b), es.call("carlson_rc", av, bv)))
            elif k == 3:
                vals.append((ek.carlson_rc(2.0, a), es.call("carlson_rc", 2.0, av)))
            elif k == 4:
                vals.append((ek.erf(a), ms.ss.unary("erf", av)))
            elif k == 5:
                vals.append((ek.hypot(a, b), ms.binary("hypot", av, bv)))
            elif k == 6:
                vals.append((ek.atan2(a, b), ms.ts.atan2(av, bv)))
            elif k == 7:
                vals.append((a * b, (av * bv).astype(f)))
            else:
                vals.append((ek.select(a < b, a, b), np.where(av < bv, av, bv)))
    return vals[3:]


@pytest.mark.parametrize("seed", range(12))
def test_random_dags_on_the_host_compiled_kernel(ek, oracle, seed):
    rng = np.random.default_rng(8800 + seed)
    n = int(rng.choice([31, 4097, 9000]))
    table = {}
    vals = _dag(ek, rng, n, table)
    keep = [vals[int(i)] for i in rng.choice(len(vals), size=min(4, len(vals)), replace=False)]
    del vals
    prog = ek.debug_program()
    before = FastKernelEmulator.native_sweeps
    emu = es.EllKernelEmulator(oracle, table, _Factory.addresses)
    emu.run(prog)
    if n > 1000:
        assert FastKernelEmulator.native_sweeps > before, "no sweep ran on the host-compiled fast kernel"
    for arr, want in keep:
        got = emu.vars[arr.index]
        ok = es.same_bits(got, np.broadcast_to(want, got.shape))
        assert ok.all(), (seed, n, got[~ok][:4], np.broadcast_to(want, got.shape)[~ok][:4])


def test_host_kernel_on_the_golden_arguments(ek, oracle):
    """every function on the arguments of ell.npz through the host-compiled kernel (ek_math.cuh compiled as host code),
    against the restatements, raw bits away from NaNs"""
    d = _golden()
    for name in NAMES:
        table = {}
        F = _Factory(ek.Float32, table, 0x7f0000000000)
        raw = (d["tx"], d["ty"], d["tz"]) if name in es.TERNARY else (d["px"], d["py"])
        args = [F.copy(a) for a in raw]
        r = getattr(ek, name)(*args)
        emu = es.EllKernelEmulator(oracle, table, _Factory.addresses)
        before = FastKernelEmulator.native_sweeps
        emu.run(ek.debug_program())
        assert FastKernelEmulator.native_sweeps == before + 1
        assert es.same_bits(emu.vars[r.index], es.call(name, *raw)).all(), name
        del r, args
        gc.collect()


# ------------------------------------------------------------------ SASS
@pytest.mark.parametrize("T", [128, 256])
@pytest.mark.parametrize("ext", [32, 63])
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
    """ek_fast_kernel<T, 32> and <T, 63>: no local-memory frame, at most 128 registers"""
    found = 0
    for block in _cuobjdump("ek_sweep_fast_trig.o", "-res-usage").split("Function ")[1:]:
        name = block.split(":")[0]
        if re.search(r"ek_fast_kernelILi(128|256)ELj(32|63)E", name):
            found += 1
            m = re.search(r"STACK:(\d+)", block)
            assert m and int(m.group(1)) == 0, (name, block[:300])
            m = re.search(r"REG:(\d+)", block)
            assert m and int(m.group(1)) <= 128, (name, block[:300])
    assert found == 4, found


# SHA-256 of the SASS instructions of the two math-set instantiations as nvcc 12.9 compiles them before and after the
# Carlson set was added: the bodies that ran them run them unchanged
PARENT_SASS_MATH = {
    "ek_fast_kernelILi128ELj16EEEv11EkSweepArgs": "85500bab822e1b8836058bc8b6f5db86c98d40abeaca12d858bf3e44d58de955",
    "ek_fast_kernelILi256ELj16EEEv11EkSweepArgs": "e070d5ffbabce6f231287bdc15650b4d27f49ac7744f04a08583bf669217de0f",
    "ek_fast_kernelILi128ELj31EEEv11EkSweepArgs": "0b9b72f2435e3d305f73ab10e95c18197ba5e575c070ebf23cba63a4913bc1b2",
    "ek_fast_kernelILi256ELj31EEEv11EkSweepArgs": "18c8f4a38e2041221d7c0529f2224b9b414f07bc7e6d867d2df5c3fa43867a99",
}


def test_kernels_of_other_programs_are_unchanged():
    if _nvcc_release() != "12.9":
        pytest.skip("the digests are of nvcc 12.9's SASS")
    fns = _functions("ek_sweep_fast_trig.o")
    for name, digest in PARENT_SASS_MATH.items():
        assert _digest(fns[name]) == digest, name
    for key, digest in PARENT_SASS.items():
        obj, name = key.split("|")
        if obj == "ek_sweep_fast_trig.o":
            assert _digest(fns[name]) == digest, name
