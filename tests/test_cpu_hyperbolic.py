"""CPU: the Float32 operations sinh, cosh, tanh, asinh, acosh, atanh and cbrt (EK_OP_SINH ... EK_OP_CBRT).  What the
planner records and lowers for them (ek_debug_program), the operations it refuses, the C restatements of
tests/hyp_oracle.c against the reference CPU path (tests/golden/hyp.npz) and against the traced bodies they replace
(tests/golden/hyp_traced.json, run on the numpy interpreter), and random expression DAGs that contain them on the numpy
interpreter and on the host-compiled fast kernel (tests/cpu_kernel), bit for bit."""
import gc
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import hyp_support as hs
from ek_emulator import Emulator
from fast_kernel_emu import FastKernelEmulator
from test_cpu_emulator import _Factory

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
UNARY = hs.UNARY
# the numbers of body instructions (of the main sweep) and of sweeps of the traced bodies (the dry run stored in
# tests/golden/hyp_traced.json)
TRACED = {"sinh": (12, 1), "cosh": (4, 1), "tanh": (19, 1), "asinh": (22, 1), "acosh": (23, 2), "atanh": (21, 1),
          "cbrt": (50, 2), "sincosh": (14, 1)}
# the largest distance to the reference CPU path, in ulps, of the functions that take rcp (rcpps + one Newton step
# there, correctly rounded here), and the arguments that take it
RCP_ULPS = {"sinh": 2, "cosh": 2, "tanh": 4}
RCP_BRANCH = {"sinh": lambda x: np.abs(x) > 1, "cosh": lambda x: np.ones(x.shape, bool),
              "tanh": lambda x: np.abs(x) >= 0.625}


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


def _traced():
    with open(os.path.join(GOLDEN, "hyp_traced.json")) as f:
        return json.load(f)


def _inputs(n, seed):
    """special values, then random bit patterns, then uniform values over the ranges where the branches change"""
    d = np.load(os.path.join(GOLDEN, "hyp.npz"))
    rng = np.random.default_rng(seed)
    r = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
    r[: n // 4] = rng.uniform(-2, 2, n // 4).astype(np.float32)
    r[n // 4: n // 2] = rng.uniform(-100, 100, n // 4).astype(np.float32)
    return np.concatenate([d["x"], r])


# ------------------------------------------------------------------ the C restatements against the reference CPU path
@pytest.mark.parametrize("name,ref", [(n, n) for n in UNARY] + [("sinh", "sincosh_s"), ("cosh", "sincosh_c")])
def test_restatement_against_hyp_golden(name, ref):
    d = np.load(os.path.join(GOLDEN, "hyp.npz"))
    x, want = d["x"], d[ref]
    got = hs.unary(name, x)
    if name not in RCP_ULPS:
        bad = _bits(got) != _bits(want)               # raw bits, NaNs included
        assert not bad.any(), (name, x[bad][:5], got[bad][:5], want[bad][:5])
        return
    # exact where no reciprocal is taken; within the rcpps + Newton bound where it is, with the same NaNs and infinities
    recip = RCP_BRANCH[name](x)
    assert (_bits(got)[~recip] == _bits(want)[~recip]).all()
    finite = recip & np.isfinite(got) & np.isfinite(want)
    assert _ulps(got[finite], want[finite]).max() <= RCP_ULPS[name]
    assert (np.isnan(got) == np.isnan(want)).all() and (np.isinf(got) == np.isinf(want)).all()
    assert (np.signbit(got) == np.signbit(want))[~np.isnan(got)].all()


def test_reference_quirks_are_reproduced():
    """cbrt(+-0) = +-0.337986261 and cbrt(1e-45) = 1.2e-13 (frexp takes 0 and denormals for normal numbers),
    acosh(x < 1) the all-ones NaN of r_small |= x1 < 0, atanh(+-1) = +-inf: the reference CPU path gives the same"""
    x = np.array([0.0, -0.0, 1e-45, -1e-45, 0.5, -3.0, 1.0 - 2 ** -24, 1.0, -1.0], np.float32)
    cb, ac, at = hs.unary("cbrt", x[:4]), hs.unary("acosh", x[4:7]), hs.unary("atanh", x[7:])
    assert list(_bits(cb)) == [0x3ead0c89, 0xbead0c89, 0x2a0775a2, 0xaa0775a2]
    assert np.float32(cb[0]) == np.float32(0.337986261) and abs(cb[2] - 1.2031221e-13) < 1e-19
    assert list(_bits(ac)) == [0xffffffff] * 3
    assert list(at) == [np.inf, -np.inf]
    d = np.load(os.path.join(GOLDEN, "hyp.npz"))
    for name, xs in (("cbrt", x[:4]), ("acosh", x[4:6]), ("atanh", x[7:])):
        for v in xs:
            k = np.flatnonzero(_bits(d["x"]) == _bits(np.float32(v)))
            assert len(k), (name, v)
            assert _bits(d[name][k[0]]) == _bits(hs.unary(name, np.array([v], np.float32)))[0], (name, v)


# ------------------------------------------------------------------ the restatements are the traced bodies
@pytest.mark.parametrize("name", list(TRACED))
def test_traced_program_equals_restatement(oracle, name):
    """The program that array_math.h's generic body records on this backend (the dry run stored in hyp_traced.json,
    recorded over a mapped CUDAArray<float> by tests/golden/ref_hyp_traced.cpp) runs on the numpy interpreter for
    about 4.2 million arguments and must give the restatement's raw bits, NaNs included."""
    t = _traced()[name]
    sweeps = t["program"]["sweeps"]
    assert len(sweeps) == TRACED[name][1]
    assert len(sweeps[-1]["body"]) == TRACED[name][0]
    x = _inputs(1 << 22, 31 + list(TRACED).index(name))
    prog = dict(t["program"], sweeps=[dict(s, n=len(x)) if s["n"] > 1 else s for s in sweeps])
    emu = Emulator(oracle, {t["x"]: x})
    emu.run(prog)
    wants = [hs.unary("sinh", x), hs.unary("cosh", x)] if name == "sincosh" else [hs.unary(name, x)]
    for out, want in zip(t["out"], wants):
        got = emu.vars[out]
        bad = _bits(got) != _bits(want)
        assert not bad.any(), (name, int(bad.sum()), x[bad][:5], _bits(got)[bad][:5], _bits(want)[bad][:5])


# ------------------------------------------------------------------ recording, lowering, instantiation
def _names(prog, instrs, fast=False):
    return [(prog["fops"] if fast else prog["ops"])[t[0]] for t in instrs]


def _arith(names):
    return [n for n in names if n not in ("NOP", "ST_32", "LOAD_32", "LOAD", "LOADU", "LD_F16", "ST_F16", "LD_U16")]


@pytest.mark.parametrize("name", list(UNARY) + ["sincosh"])
def test_each_function_is_one_node_and_one_instruction(ek, name):
    table = {}
    F = _Factory(ek.Float32, table, 0x7f0000000000)
    x = F.copy(np.ones(1 << 20, np.float32))
    r = ek.sincosh(x) if name == "sincosh" else (getattr(ek, name)(x),)
    want = ["SINH_F32", "COSH_F32"] if name == "sincosh" else [name.upper() + "_F32"]
    plan = ek.debug_plan()
    assert plan.count("\n  body ") == len(want), plan
    assert plan.count("sweep ") == 1, "a second launch: " + plan          # acosh and cbrt traced needed two
    prog = ek.debug_program()
    (sw,) = prog["sweeps"]
    assert _arith(_names(prog, sw["body"])) == want
    assert sw["config"]["fast"] == 1
    assert _arith(_names(prog, sw["fast"]["body"], fast=True)) == want
    assert sw["fast"]["ext"] == 4, "the launcher would not pick the hyperbolic instantiation"
    del r


def test_float16_storage_with_tanh_needs_both_sets(ek):
    """(the launcher runs such a body, like any with more than one optional set but Float16 + trigonometric, on
    ek_fast_kernel<T, EK_FX_ALL>)"""
    table = {}
    H = _Factory(ek.Float16, table, 0x7c0000000000)
    x = ek.Float32(H.copy(np.ones(1 << 16, np.float16)))
    r = ek.Float16(ek.tanh(x) + ek.cbrt(x))
    prog = ek.debug_program()
    (sw,) = prog["sweeps"]
    fast = _names(prog, sw["fast"]["body"], fast=True)
    assert fast[0] == "LD_F16" and fast[-1] == "ST_F16" and "TANH_F32" in fast and "CBRT_F32" in fast, fast
    assert sw["config"]["fast"] == 1 and sw["fast"]["ext"] == 5
    del r


@pytest.mark.parametrize("name", UNARY)
@pytest.mark.parametrize("cls,tname", [("Float64", "f64"), ("Int32", "i32"), ("UInt32", "u32")])
def test_other_types_are_refused(ek, name, cls, tname):
    table = {}
    F = _Factory(getattr(ek, cls), table, 0x7b0000000000)
    a = F.copy(np.ones(4096, {"Float64": np.float64, "Int32": np.int32, "UInt32": np.uint32}[cls]))
    r = getattr(ek, name)(a)
    with pytest.raises(ek.EnokiError) as e:
        ek.debug_plan()
    assert f"op {name} not supported for type {tname}" in str(e.value), str(e.value)
    del r


@pytest.mark.parametrize("name", UNARY)
def test_float16_is_refused(ek, name):
    table = {}
    a = _Factory(ek.Float16, table, 0x7c0000000000).copy(np.ones(4096, np.float16))
    r = getattr(ek, name)(a)
    with pytest.raises(ek.EnokiError) as e:
        ek.debug_plan()
    assert f"op {name} is not supported on Float16" in str(e.value), str(e.value)
    del r


def test_opcodes_are_appended(ek):
    assert [ek.OP[n.upper()] for n in UNARY] == list(range(ek.OP["ATAN2"] + 1, ek.OP["ATAN2"] + 8))
    assert len(ek._OPS) == ek.OP["CBRT"] + 1


# ------------------------------------------------------------------ random DAGs: interpreter and host-compiled kernel
def _dag(ek, rng, n, table):
    """A random Float32 DAG mixing the seven functions (and atan2 / tan from the trigonometric set) with add / mul /
    select; returns [(array, expected numpy value)]"""
    F = _Factory(ek.Float32, table, 0x7f0000000000)
    vals = []
    for _ in range(3):
        x = rng.uniform(-3, 3, n).astype(np.float32)
        x[rng.integers(0, n, max(n // 50, 1))] = rng.choice(np.array([0.0, -0.0, 1.0, -1.0, 0.5, 1e10, np.inf, -np.inf,
                                                                      np.nan, 1e-45, 100.0], np.float32))
        vals.append((F.copy(x), x))
    with np.errstate(all="ignore"):
        for _ in range(int(rng.integers(6, 16))):
            k = int(rng.integers(0, 11))
            (a, av), (b, bv) = (vals[int(i)] for i in rng.integers(0, len(vals), 2))
            if k < 7:
                vals.append((getattr(ek, UNARY[k])(a), hs.unary(UNARY[k], np.broadcast_to(av, (n,)))))
            elif k == 7:
                vals.append((ek.atan2(a, b), hs.ts.atan2(av, bv)))
            elif k == 8:
                vals.append((a * b, (av * bv).astype(np.float32)))
            elif k == 9:
                vals.append((a + 0.5, (av + np.float32(0.5)).astype(np.float32)))
            else:
                vals.append((ek.select(a < b, a, b), np.where(av < bv, av, bv)))
    return vals[3:]


def _dag_case(ek, oracle, seed, emulator):
    rng = np.random.default_rng(8800 + seed)
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
        ok = hs.same_bits(got, np.broadcast_to(want, got.shape))
        assert ok.all(), (seed, n, got[~ok][:4], np.broadcast_to(want, got.shape)[~ok][:4])
    assert red.index in emu.vars
    return n


@pytest.mark.parametrize("form", ["assembled", "lowered"])
@pytest.mark.parametrize("seed", range(30))
def test_random_hyp_dags_on_the_interpreter(ek, oracle, seed, form):
    hs.HypEmulator.prefer_fast = form == "lowered"
    try:
        _dag_case(ek, oracle, seed, hs.HypEmulator)
    finally:
        hs.HypEmulator.prefer_fast = False


@pytest.mark.parametrize("seed", range(30))
def test_random_hyp_dags_on_the_host_compiled_kernel(ek, oracle, seed):
    before = FastKernelEmulator.native_sweeps
    n = _dag_case(ek, oracle, seed, hs.HypKernelEmulator)
    if n > 1000:
        assert FastKernelEmulator.native_sweeps > before, "no sweep ran on the host-compiled fast kernel"


def test_random_hyp_dags_on_the_128_thread_kernel():
    """The host-compiled kernel once more restricted to T = 128 (EK_FAST_T is read once per process: a child process)."""
    env = dict(os.environ, EK_FAST_T="128")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_cpu_hyperbolic.py"), "-q", "-x",
                        "-k", "host_compiled_kernel", "-p", "no:cacheprovider"], capture_output=True, text=True,
                       timeout=1800, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout


def test_host_kernel_on_the_golden_arguments(ek, oracle):
    """every function on the arguments of hyp.npz (specials, branch thresholds, random values) through the
    host-compiled kernel, against the restatements, raw bits"""
    x = np.load(os.path.join(GOLDEN, "hyp.npz"))["x"]
    for name in UNARY:
        table = {}
        r = getattr(ek, name)(_Factory(ek.Float32, table, 0x7f0000000000).copy(x))
        emu = hs.HypKernelEmulator(oracle, table, _Factory.addresses)
        before = FastKernelEmulator.native_sweeps
        emu.run(ek.debug_program())
        assert FastKernelEmulator.native_sweeps == before + 1
        got = emu.vars[r.index]
        want = hs.unary(name, x)
        assert hs.same_bits(got, want).all(), name
        ok = ~np.isnan(want)                              # the host kernel's NaNs follow its own operand order
        assert (_bits(got)[ok] == _bits(want)[ok]).all(), name
        del r
        gc.collect()


# ------------------------------------------------------------------ SASS
@pytest.mark.parametrize("T", [128, 256])
@pytest.mark.parametrize("ext", [4, 7])
def test_dispatch_frames_have_no_accumulator_copies(T, ext):
    """the check of tests/test_cpu_trig.py on the instantiations that carry the hyperbolic operations"""
    from test_cpu_trig import _sass_of
    sass = _sass_of("ek_sweep_fast_trig.o", f"14ek_fast_kernelILi{T}ELj{ext}EEEv11EkSweepArgs")
    fetch = [i for i, l in enumerate(sass) if re.match(r"LDC\.64 R\d+, c\[0x0\]\[R\d+\+0x21[08]\]", l)]
    start = next((i for i in fetch if sum(1 for l in sass[i:i + 40] if re.match(r"@P\d LDS\.128", l)) >= 8), None)
    assert start is not None, "hot-loop fetch not found"
    frame = sass[max(start - 4, 0):start + 45]
    moves = [l for l in frame if re.match(r"(IMAD\.MOV\.U32|MOV) R\d+, (RZ, RZ, )?R\d+", l)]
    assert len(moves) <= 2, "ptxas copies the accumulator in the dispatch frame:\n" + "\n".join(frame)
