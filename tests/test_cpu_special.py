"""CPU: the Float32 operations erf, erfc, erfinv, lgamma and tgamma (EK_OP_ERF ... EK_OP_TGAMMA).  What the planner
records and lowers for them (ek_debug_program), the operations it refuses, the C restatements of tests/special_oracle.c
against the reference CPU path (tests/golden/special.npz) and against the traced bodies they replace
(tests/golden/special_traced.json, run on the numpy interpreter), random expression DAGs that contain them on the numpy
interpreter and on the host-compiled fast kernel (tests/cpu_kernel), bit for bit, and the SASS of the kernels that carry
them (and of those that must not change)."""
import gc
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

import special_support as ss
from ek_emulator import Emulator
from fast_kernel_emu import FastKernelEmulator
from test_cpu_emulator import _Factory

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CSRC = os.path.join(ROOT, "enoki_b200", "csrc")
UNARY = ss.UNARY
# the number of body instructions of the traced bodies (one sweep each: the dry run stored in
# tests/golden/special_traced.json); "normal" is sqrt(2) * erfinv(2u - 1), the sampling step of the reference's
# tests/histogram.cpp
TRACED = {"erf": 46, "erfc": 46, "erfinv": 35, "lgamma": 41, "tgamma": 42, "normal": 38}
# the largest distance to the reference CPU path, in ulps, of erf and erfc where they take rcp(|x|) (rcpps + one Newton
# step there, correctly rounded here): |x| > 1 for erf, |x| >= 1 for erfc
RCP_ULPS = {"erf": 2, "erfc": 4}
RCP_BRANCH = {"erf": lambda x: np.abs(x) > 1, "erfc": lambda x: np.abs(x) >= 1}


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


def _golden():
    return np.load(os.path.join(GOLDEN, "special.npz"))


def _traced():
    with open(os.path.join(GOLDEN, "special_traced.json")) as f:
        return json.load(f)


def _inputs(n, seed):
    """special values, then random bit patterns, then uniform values over the ranges where the branches change"""
    rng = np.random.default_rng(seed)
    r = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
    r[: n // 4] = rng.uniform(-3, 3, n // 4).astype(np.float32)
    r[n // 4: n // 2] = rng.uniform(-1, 1, n // 4).astype(np.float32)
    r[n // 2: 5 * n // 8] = rng.uniform(-40, 40, n // 8).astype(np.float32)
    return np.concatenate([_golden()["x"], r])


def normal(u):
    """sqrt(2) * erfinv(2u - 1) as the restatement computes it (float32 steps)"""
    f = np.float32
    with np.errstate(all="ignore"):
        t = ((f(2) * u).astype(f) - f(1)).astype(f)
        return (ss.unary("erfinv", t) * f(np.sqrt(2.0))).astype(f)


# ------------------------------------------------------------------ the C restatements against the reference CPU path
@pytest.mark.parametrize("name", UNARY)
def test_restatement_against_special_golden(name):
    d = _golden()
    x, want = d["x"], d[name]
    got = ss.unary(name, x)
    if name not in RCP_ULPS:
        # raw bits; erfinv's NaNs included.  lgamma and tgamma of a NaN argument: the CPU path adds its all-ones NaN
        # log(sum) first, where the recorded program adds the product that carries the argument's NaN first
        keep = np.ones(x.shape, bool) if name == "erfinv" else ~np.isnan(x)
        bad = (_bits(got) != _bits(want)) & keep
        assert not bad.any(), (name, x[bad][:5], got[bad][:5], want[bad][:5])
        assert (np.isnan(got) == np.isnan(want)).all()
        return
    # exact where no reciprocal is taken; within the rcpps + Newton bound where it is, with the same NaNs and infinities
    recip = RCP_BRANCH[name](x)
    assert (_bits(got)[~recip] == _bits(want)[~recip]).all()
    finite = recip & np.isfinite(got) & np.isfinite(want)
    assert _ulps(got[finite], want[finite]).max() == RCP_ULPS[name]
    assert (np.isnan(got) == np.isnan(want)).all() and (np.isinf(got) == np.isinf(want)).all()
    assert (np.signbit(got) == np.signbit(want))[~np.isnan(got)].all()


def test_reference_edge_values_are_reproduced():
    """What special.h computes at its edges, reproduced as it is, not as it should be: erfinv(+-1) is NaN (w = +inf and
    the polynomial in sqrt(w) - 3 meets inf - inf), as is erfinv(|x| > 1); lgamma(2) is 2.4e-7; lgamma and tgamma are
    +inf at 0, -0, the negative integers and -inf, and NaN at +inf; tgamma overflows to +inf by x = 35.  The reference
    CPU path gives the same values."""
    inf, nan = np.inf, np.nan
    cases = {
        "erfinv": ([1.0, -1.0, 1.5, -2.0, inf, 0.0, -0.0, 0.99999994], [nan, nan, nan, nan, nan, 0.0, -0.0, 3.8325064]),
        "erf": ([inf, -inf, 0.0, -0.0, 10.0, 1.0, -1.0], [1.0, -1.0, 0.0, -0.0, 1.0, 0.84270066, -0.84270066]),
        "erfc": ([inf, -inf, 0.0, 10.0, -10.0, 1.0], [0.0, 2.0, 1.0, 0.0, 2.0, 0.15729924]),
        "lgamma": ([0.0, -0.0, -1.0, -2.0, -40.0, -inf, inf, 1.0, 2.0, -0.5],
                   [inf, inf, inf, inf, inf, inf, nan, 0.0, 2.3841858e-07, 1.2655122]),
        "tgamma": ([0.0, -0.0, -1.0, -7.0, -inf, inf, 35.0, 35.5, 1.0, 4.0, -0.5],
                   [inf, inf, inf, inf, inf, nan, inf, inf, 1.0, 6.0, 3.544908]),
    }
    d = _golden()
    for name, (xs, wants) in cases.items():
        x = np.array(xs, np.float32)
        got = ss.unary(name, x)
        for v, g, w in zip(x, got, np.array(wants, np.float32)):
            assert ss.same_bits(g, w), (name, v, g, w)
            k = np.flatnonzero(_bits(d["x"]) == _bits(v))
            assert len(k), (name, v)
            assert ss.same_bits(d[name][k[0]], g), (name, v, d[name][k[0]], g)


# ------------------------------------------------------------------ the restatements are the traced bodies
@pytest.mark.parametrize("name", list(TRACED))
def test_traced_program_equals_restatement(oracle, name):
    """The program that special.h's generic body records on this backend (the dry run stored in special_traced.json,
    recorded over a mapped CUDAArray<float> by tests/golden/ref_special_traced.cpp) runs on the numpy interpreter for
    about 4.2 million arguments and must give the restatement's raw bits, NaNs included."""
    t = _traced()[name]
    (sweep,) = t["program"]["sweeps"]
    assert len(sweep["body"]) == TRACED[name]
    x = _inputs(1 << 22, 41 + list(TRACED).index(name))
    if name == "normal":
        x[len(x) // 2:] = np.random.default_rng(7).uniform(0, 1, len(x) - len(x) // 2).astype(np.float32)
    prog = dict(t["program"], sweeps=[dict(sweep, n=len(x))])
    emu = Emulator(oracle, {t["x"]: x})
    emu.run(prog)
    got = emu.vars[t["out"][0]]
    want = normal(x) if name == "normal" else ss.unary(name, x)
    bad = _bits(got) != _bits(want)
    assert not bad.any(), (name, int(bad.sum()), x[bad][:5], _bits(got)[bad][:5], _bits(want)[bad][:5])


# ------------------------------------------------------------------ recording, lowering, instantiation
def _names(prog, instrs, fast=False):
    return [(prog["fops"] if fast else prog["ops"])[t[0]] for t in instrs]


def _arith(names):
    return [n for n in names if n not in ("NOP", "ST_32", "LOAD_32", "LOAD", "LOADU", "LD_F16", "ST_F16", "LD_U16")]


@pytest.mark.parametrize("name", UNARY)
def test_each_function_is_one_node_and_one_instruction(ek, name):
    table = {}
    x = _Factory(ek.Float32, table, 0x7f0000000000).copy(np.ones(1 << 20, np.float32))
    r = getattr(ek, name)(x)
    want = [name.upper() + "_F32"]
    plan = ek.debug_plan()
    assert plan.count("\n  body ") == 1, plan
    assert plan.count("sweep ") == 1, plan
    prog = ek.debug_program()
    (sw,) = prog["sweeps"]
    assert _arith(_names(prog, sw["body"])) == want
    assert sw["config"]["fast"] == 1
    assert _arith(_names(prog, sw["fast"]["body"], fast=True)) == want
    assert sw["fast"]["ext"] == 8, "the launcher would not pick the special-function instantiation"
    del r


def test_normal_sampling_step_is_one_sweep_of_four_instructions(ek):
    """sqrt(2) * erfinv(2u - 1): 38 body instructions traced, four native"""
    table = {}
    u = _Factory(ek.Float32, table, 0x7f0000000000).copy(np.full(1 << 20, 0.25, np.float32))
    r = ek.erfinv(u * 2.0 - 1.0) * float(np.float32(np.sqrt(2.0)))
    prog = ek.debug_program()
    (sw,) = prog["sweeps"]
    assert _arith(_names(prog, sw["body"]))[-2:] == ["ERFINV_F32", "MUL_F32"]
    assert len(_arith(_names(prog, sw["body"]))) == 4
    assert sw["config"]["fast"] == 1 and sw["fast"]["ext"] == 8
    del r


@pytest.mark.parametrize("mix,ext", [("tanh", 4), ("tanh+erf", 12), ("tan+lgamma", 10), ("f16+erfc", 9)])
def test_the_launcher_picks_the_smallest_instantiation(ek, mix, ext):
    """ek_fast_ext, the operation sets of the lowered body: a hyperbolic body is still EK_FX_HYP alone (4, run by
    <T, EK_FX_HYP>; mixed with Float16 storage or trigonometric operations it still runs <T, 7>); a body that mixes the
    special functions (8) with another set is run by <T, EK_FX_ALL> (15)."""
    table = {}
    if mix.startswith("f16"):
        H = _Factory(ek.Float16, table, 0x7c0000000000)
        x = ek.Float32(H.copy(np.ones(1 << 16, np.float16)))
        r = ek.Float16(ek.erfc(x))
    else:
        x = _Factory(ek.Float32, table, 0x7f0000000000).copy(np.ones(1 << 16, np.float32))
        r = {"tanh": lambda: ek.tanh(x), "tanh+erf": lambda: ek.tanh(x) + ek.erf(x),
             "tan+lgamma": lambda: ek.tan(x) * ek.lgamma(x)}[mix]()
    prog = ek.debug_program()
    (sw,) = prog["sweeps"]
    assert sw["config"]["fast"] == 1
    assert sw["fast"]["ext"] == ext, (mix, sw["fast"]["ext"])
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
    """after the hyperbolic operations, which keep their numbers after ATAN2"""
    hyp = ("SINH", "COSH", "TANH", "ASINH", "ACOSH", "ATANH", "CBRT")
    assert [ek.OP[n] for n in hyp] == list(range(ek.OP["ATAN2"] + 1, ek.OP["ATAN2"] + 8))
    assert [ek.OP[n.upper()] for n in UNARY] == list(range(ek.OP["CBRT"] + 1, ek.OP["CBRT"] + 6))
    assert ek._OPS_SPECIAL == [n.upper() for n in UNARY] and len(ek.OP) == ek.OP["TGAMMA"] + 1


# ------------------------------------------------------------------ random DAGs: interpreter and host-compiled kernel
def _dag(ek, rng, n, table):
    """A random Float32 DAG mixing the five functions (and tanh / atan2 from the other sets) with add / mul / select;
    returns [(array, expected numpy value)]"""
    F = _Factory(ek.Float32, table, 0x7f0000000000)
    vals = []
    for _ in range(3):
        x = rng.uniform(-3, 3, n).astype(np.float32)
        x[rng.integers(0, n, max(n // 50, 1))] = rng.choice(np.array([0.0, -0.0, 1.0, -1.0, 2.0, 0.5, -3.0, 1e10, np.inf,
                                                                      -np.inf, np.nan, 1e-45, 36.0], np.float32))
        vals.append((F.copy(x), x))
    with np.errstate(all="ignore"):
        for _ in range(int(rng.integers(6, 16))):
            k = int(rng.integers(0, 10))
            (a, av), (b, bv) = (vals[int(i)] for i in rng.integers(0, len(vals), 2))
            if k < 5:
                vals.append((getattr(ek, UNARY[k])(a), ss.unary(UNARY[k], np.broadcast_to(av, (n,)))))
            elif k == 5:
                vals.append((ek.tanh(a), ss.hs.unary("tanh", np.broadcast_to(av, (n,)))))
            elif k == 6:
                vals.append((ek.atan2(a, b), ss.ts.atan2(av, bv)))
            elif k == 7:
                vals.append((a * b, (av * bv).astype(np.float32)))
            elif k == 8:
                vals.append((a + 0.5, (av + np.float32(0.5)).astype(np.float32)))
            else:
                vals.append((ek.select(a < b, a, b), np.where(av < bv, av, bv)))
    return vals[3:]


def _dag_case(ek, oracle, seed, emulator):
    rng = np.random.default_rng(9900 + seed)
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
        ok = ss.same_bits(got, np.broadcast_to(want, got.shape))
        assert ok.all(), (seed, n, got[~ok][:4], np.broadcast_to(want, got.shape)[~ok][:4])
    assert red.index in emu.vars
    return n


@pytest.mark.parametrize("form", ["assembled", "lowered"])
@pytest.mark.parametrize("seed", range(30))
def test_random_special_dags_on_the_interpreter(ek, oracle, seed, form):
    ss.SpecEmulator.prefer_fast = form == "lowered"
    try:
        _dag_case(ek, oracle, seed, ss.SpecEmulator)
    finally:
        ss.SpecEmulator.prefer_fast = False


@pytest.mark.parametrize("seed", range(30))
def test_random_special_dags_on_the_host_compiled_kernel(ek, oracle, seed):
    before = FastKernelEmulator.native_sweeps
    n = _dag_case(ek, oracle, seed, ss.SpecKernelEmulator)
    if n > 1000:
        assert FastKernelEmulator.native_sweeps > before, "no sweep ran on the host-compiled fast kernel"


def test_random_special_dags_on_the_128_thread_kernel():
    """The host-compiled kernel once more restricted to T = 128 (EK_FAST_T is read once per process: a child process)."""
    env = dict(os.environ, EK_FAST_T="128")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_cpu_special.py"), "-q", "-x",
                        "-k", "host_compiled_kernel", "-p", "no:cacheprovider"], capture_output=True, text=True,
                       timeout=1800, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout


def test_host_kernel_on_the_golden_arguments(ek, oracle):
    """every function on the arguments of special.npz (specials, branch thresholds, random values) through the
    host-compiled kernel, against the restatements, raw bits away from NaNs"""
    x = _golden()["x"]
    for name in UNARY:
        table = {}
        r = getattr(ek, name)(_Factory(ek.Float32, table, 0x7f0000000000).copy(x))
        emu = ss.SpecKernelEmulator(oracle, table, _Factory.addresses)
        before = FastKernelEmulator.native_sweeps
        emu.run(ek.debug_program())
        assert FastKernelEmulator.native_sweeps == before + 1
        got = emu.vars[r.index]
        want = ss.unary(name, x)
        assert ss.same_bits(got, want).all(), name
        ok = ~np.isnan(want)                              # the host kernel's NaNs follow its own operand order
        assert (_bits(got)[ok] == _bits(want)[ok]).all(), name
        del r
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
@pytest.mark.parametrize("ext", [8, 15])
def test_dispatch_frames_have_no_accumulator_copies(T, ext):
    """the check of tests/test_cpu_trig.py on the instantiations that carry the special functions"""
    from test_cpu_trig import _sass_of
    sass = _sass_of("ek_sweep_fast_trig.o", f"14ek_fast_kernelILi{T}ELj{ext}EEEv11EkSweepArgs")
    fetch = [i for i, l in enumerate(sass) if re.match(r"LDC\.64 R\d+, c\[0x0\]\[R\d+\+0x21[08]\]", l)]
    start = next((i for i in fetch if sum(1 for l in sass[i:i + 40] if re.match(r"@P\d LDS\.128", l)) >= 8), None)
    assert start is not None, "hot-loop fetch not found"
    frame = sass[max(start - 4, 0):start + 45]
    moves = [l for l in frame if re.match(r"(IMAD\.MOV\.U32|MOV) R\d+, (RZ, RZ, )?R\d+", l)]
    assert len(moves) <= 2, "ptxas copies the accumulator in the dispatch frame:\n" + "\n".join(frame)


def test_instantiations_carrying_the_special_functions_use_no_stack():
    """ek_fast_kernel<T, 8>, <T, 15> and ek_sweep_kernel<V, INLINE, true>: no local-memory frame"""
    for obj, pat in (("ek_sweep_fast_trig.o", r"ek_fast_kernelILi(128|256)ELj(8|15)E"),
                     ("ek_sweep_trig.o", r"ek_sweep_kernelILi[48]ELb[01]ELb1E")):
        found = 0
        for block in _cuobjdump(obj, "-res-usage").split("Function ")[1:]:
            name = block.split(":")[0]
            if re.search(pat, name):
                found += 1
                m = re.search(r"STACK:(\d+)", block)
                assert m and int(m.group(1)) == 0, (name, block[:300])
        assert found == 4, (obj, found)


# SHA-256 of the SASS instructions of every kernel that programs without the special functions run, as nvcc 12.9
# compiles this repository before and after they were added: ek_sweep.o and ek_sweep_fast.o whole, and the
# trigonometric, Float16 + trigonometric, hyperbolic and Float16 + trigonometric + hyperbolic instantiations of the fast
# kernel
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
    "ek_sweep_fast_trig.o|ek_fast_kernelILi256ELj2EEEv11EkSweepArgs":
        "f4e7cf59785c2582843d9e7f4a874a91bdf5b976b591183d71f8f089a26fff5c",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi256ELj3EEEv11EkSweepArgs":
        "f167adf330ab54a721463ae7e694981d7acdb3da8848a4953e92d86a48a2947d",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi256ELj4EEEv11EkSweepArgs":
        "0f734899cdbc077ab21c152ff1ce5c77d6fff9c31bb7bd2a8553e3c4c4639a4e",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi128ELj7EEEv11EkSweepArgs":
        "6981518b309e3379b9c66b9bd92f607a73840959f17039ee4f62467be9fed16b",
    "ek_sweep_fast_trig.o|ek_fast_kernelILi256ELj7EEEv11EkSweepArgs":
        "d7b0253e8fe26ca093a3836400b0c8974b6486a0c2709cfd760b1e200512cfec",
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
    were added to the trigonometric instantiations); these kernels compile to the same instructions as before the
    special functions existed."""
    if _nvcc_release() != "12.9":
        pytest.skip("the digests are of nvcc 12.9's SASS")
    want = {k.split("|")[1]: v for k, v in PARENT_SASS.items() if k.split("|")[0] == obj}
    fns = _functions(obj)
    assert want and set(want) <= set(fns)
    for name, digest in want.items():
        assert _digest(fns[name]) == digest, name
