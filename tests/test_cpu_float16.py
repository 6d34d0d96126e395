"""CPU: Float16 arrays as a storage format.  What the assembler plans and lowers for them (ek_debug_program), the numpy
interpreter (tests/ek_emulator.py, taught the two Float16 conversions below) on the assembler's programs and the
host-compiled fast kernel (tests/cpu_kernel) on the lowered ones, bit for bit against numpy's float16 (IEEE binary16,
round to nearest even), and the operations that stay rejected."""
import gc

import numpy as np
import pytest

import fast_kernel_emu
from ek_emulator import Emulator
from fast_kernel_emu import FastKernelEmulator
from test_cpu_emulator import _Factory


def _f16_cvt(name, R):
    """CVT_F32_F16 (round to nearest even) and CVT_F16_F32 (exact) on the accumulator's bits; None for other names."""
    if name == "CVT_F32_F16":
        with np.errstate(over="ignore"):
            return R.view(np.float32).astype(np.float16).view(np.uint16).astype(np.uint32)
    if name == "CVT_F16_F32":
        return (R & np.uint32(0xffff)).astype(np.uint16).view(np.float16).astype(np.float32).view(np.uint32)
    return None


class F16Emulator(Emulator):
    def _exec64(self, name, imm, R, Rh, B, Bh, C, Ch, staged, cb):
        r = _f16_cvt(name, R)
        return (r, Rh) if r is not None else super()._exec64(name, imm, R, Rh, B, Bh, C, Ch, staged, cb)


class F16KernelEmulator(FastKernelEmulator):
    """Fast sweeps on the host-compiled kernel, the others on the interpreter above."""
    def _exec64(self, name, imm, R, Rh, B, Bh, C, Ch, staged, cb):
        r = _f16_cvt(name, R)
        return (r, Rh) if r is not None else super()._exec64(name, imm, R, Rh, B, Bh, C, Ch, staged, cb)


@pytest.fixture(autouse=True)
def clean_trace(ek, monkeypatch):
    monkeypatch.setitem(fast_kernel_emu._DT, ek.EK_FLOAT16, np.float16)     # Float16 outputs of the host-compiled kernel
    gc.collect()
    yield
    gc.collect()
    ek.lib().ek_debug_discard_side_effects()
    gc.collect()


def _halves(rng, n, lo=-4.0, hi=4.0):
    return rng.uniform(lo, hi, n).astype(np.float16)


def _run(prog, oracle, table, form):
    """Executes `prog`: the assembler's form on the interpreter, or the lowered form on the host-compiled fast kernel."""
    data = {k: np.array(v, copy=True) for k, v in table.items()}
    if form == "kernel":
        emu = F16KernelEmulator(oracle, data, _Factory.addresses)
        before = FastKernelEmulator.native_sweeps
        emu.run(prog)
        assert FastKernelEmulator.native_sweeps > before, "no sweep ran on the host-compiled fast kernel"
        return emu
    emu = F16Emulator(oracle, data, _Factory.addresses)
    emu.run(prog)
    return emu


def _names(prog, instrs, fast=False):
    return [(prog["fops"] if fast else prog["ops"])[t[0]] for t in instrs]


def _c2_f16(ek, table, xs):
    """C2 (bench.py) with Float16 storage: four Float16 inputs widened to Float32, the Float32 expression, the result
    rounded to Float16.  Built in its own frame so that the Float32 temporaries are not kept as outputs."""
    F = _Factory(ek.Float16, table, 0x7c0000000000)
    x0, x1, x2, x3 = (ek.Float32(F.copy(x)) for x in xs)
    t = ek.fmadd(x0, x1, x2)
    return ek.Float16(ek.fmadd(ek.sin(ek.fmadd(x3, ek.exp(-(t * t)), x0)), x1, ek.sqrt(abs(t))))


def _c2_ref(oracle, P, xs):
    f = [np.ascontiguousarray(x.astype(np.float32)) for x in xs]
    want = np.zeros(len(f[0]), np.float32)
    oracle.or_c2(P(f[0]), P(f[1]), P(f[2]), P(f[3]), P(want), np.uint64(len(want)).item())
    return want.astype(np.float16)


@pytest.mark.parametrize("n", [4097, 20_011])
def test_c2_with_float16_storage_lowers_to_the_fused_fast_forms(ek, oracle, P, n):
    rng = np.random.default_rng(n)
    xs = [_halves(rng, n) for _ in range(4)]
    table = {}
    out = _c2_f16(ek, table, xs)
    prog = ek.debug_program()
    (sw,) = prog["sweeps"]
    body = _names(prog, sw["body"])
    assert body.count("LD_U16") == 4 and body.count("CVT_F16_F32") == 4
    assert body[-2:] == ["CVT_F32_F16", "ST_16"]
    assert sw["config"]["fast"] == 1
    fast = _names(prog, sw["fast"]["body"], fast=True)
    assert fast.count("LD_F16") == 4 and fast[-1] == "ST_F16"
    assert not any(f in ("LD_U16", "CVT_F16_F32", "CVT_F32_F16", "ST_16") for f in fast)
    assert [s[2] for s in sw["staged"]] == [2, 2, 2, 2]
    want = _c2_ref(oracle, P, xs)
    for form in ("assembled", "kernel"):
        got = _run(prog, oracle, table, form).vars[out.index]
        assert got.itemsize == 2 and got.shape == (n,), (form, got.dtype, got.shape)
        bad = got.view(np.uint16) != want.view(np.uint16)
        assert not bad.any(), (form, int(bad.sum()), got[bad][:4], want[bad][:4])


def test_float32_to_float16_rounding_on_the_host_compiled_kernel(ek, oracle):
    """Every rounding boundary of binary16 through FOP_ST_F16 (the host build of the kernel's conversion) and through
    the interpreter, against numpy (NaN payloads are not compared)."""
    h = np.arange(0x7c00, dtype=np.uint32)                       # every finite non-negative half
    up = np.concatenate([h[1:], [0x7c00]])
    lo = (h.astype(np.uint16).view(np.float16).astype(np.float32)).view(np.uint32)
    hi = (up.astype(np.uint16).view(np.float16).astype(np.float32)).view(np.uint32)
    mid = (lo.astype(np.uint64) + hi) // 2                          # the f32 midpoint between neighbours (exact)
    cases = np.concatenate([mid - 1, mid, mid + 1, lo, [0x477fe000, 0x477ff000, 0x477fefff, 0x7f800000, 0x7f7fffff, 1, 0x00800000,
                                                          0x33000000, 0x33000001, 0x32ffffff]]).astype(np.uint32)
    cases = np.concatenate([cases, cases | np.uint32(0x80000000)])
    x = cases.view(np.float32)
    table = {}
    F = _Factory(ek.Float32, table, 0x7b0000000000)
    out = ek.Float16(F.copy(x))
    prog = ek.debug_program()
    assert _names(prog, prog["sweeps"][0]["fast"]["body"], fast=True)[-1] == "ST_F16"
    with np.errstate(over="ignore"):
        want = x.astype(np.float16).view(np.uint16)
    for form in ("assembled", "kernel"):
        got = _run(prog, oracle, table, form).vars[out.index].view(np.uint16)
        bad = got != want
        assert not bad.any(), (form, int(bad.sum()), cases[bad][:4], got[bad][:4], want[bad][:4])


def test_every_half_to_float32_on_the_host_compiled_kernel(ek, oracle):
    h = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    h = h[~np.isnan(h.view(np.float16))]
    table = {}
    F = _Factory(ek.Float16, table, 0x7b8000000000)
    out = ek.Float32(F.copy(h.view(np.float16)))
    prog = ek.debug_program()
    assert _names(prog, prog["sweeps"][0]["fast"]["body"], fast=True)[0] == "LD_F16"
    want = h.view(np.float16).astype(np.float32).view(np.uint32)
    for form in ("assembled", "kernel"):
        got = _run(prog, oracle, table, form).vars[out.index].view(np.uint32)
        assert (got == want).all(), form


def test_select_and_bitcast_stay_on_the_general_kernel(ek, oracle):
    n = 5000
    rng = np.random.default_rng(1)
    a, b = _halves(rng, n), _halves(rng, n, -60000, 60000)
    m = rng.integers(0, 2, n).astype(np.bool_)
    bits = rng.integers(0, 1 << 16, n).astype(np.uint16)
    table = {}
    F16 = _Factory(ek.Float16, table, 0x7c0000000000)
    fa, fb = F16.copy(a), F16.copy(b)
    fm = _Factory(ek.Mask, table, 0x7d0000000000).copy(m)
    fu = _Factory(ek.UInt16, table, 0x7e0000000000).copy(bits)
    sel = ek.select(fm, fa, fb)
    as_f16 = ek.reinterpret(ek.Float16, fu)
    as_i32 = ek.Int32(ek.reinterpret(ek.Int16, fb))          # Float16 bits re-extended as Int16, then widened
    lit = ek.select(fm, ek.Float16(1.0 + 2.0 ** -11 + 2.0 ** -30), fa)    # literal: half(float(x)), 0x3c00
    prog = ek.debug_program()
    (sw,) = prog["sweeps"]
    assert sw["config"]["fast"] == 0 and "fast" not in sw
    body = _names(prog, sw["body"])
    assert "SEXT16" in body and "ST_16" in body
    assert 0x3C00 in sw["lits"]
    emu = _run(prog, oracle, table, "assembled")
    assert (emu.vars[sel.index].view(np.uint16) == np.where(m, a, b).view(np.uint16)).all()
    assert (emu.vars[as_f16.index].view(np.uint16) == bits).all()
    assert (emu.vars[as_i32.index].view(np.int32) == b.view(np.int16).astype(np.int32)).all()
    assert (emu.vars[lit.index].view(np.uint16) == np.where(m, np.uint16(0x3C00), a.view(np.uint16))).all()


def test_float64_to_float16_goes_through_float32(ek, oracle):
    x = np.array([1 + 2.0 ** -11 + 2.0 ** -30, 65519.99, 65520.0, 2.0 ** -25, 2.0 ** -25 * (1 + 2.0 ** -40), -0.0, 1e300,
                  3.14159265358979] * 700, np.float64)
    table = {}
    out = ek.Float16(_Factory(ek.Float64, table, 0x7c0000000000).copy(x))
    prog = ek.debug_program()
    (sw,) = prog["sweeps"]
    body = _names(prog, sw["body"])
    assert body[-3:] == ["CVT_F64_F32", "CVT_F32_F16", "ST_16"], body
    got = _run(prog, oracle, table, "assembled").vars[out.index].view(np.uint16)
    with np.errstate(over="ignore"):
        want = x.astype(np.float32).astype(np.float16).view(np.uint16)
    assert got[0] == 0x3C00 and x[:1].astype(np.float16).view(np.uint16)[0] == 0x3C01     # a single rounding differs
    assert (got == want).all()


@pytest.mark.parametrize("target", ["Int32", "UInt32", "Int8", "Float64"])
def test_float16_to_other_types_goes_through_float32(ek, oracle, target):
    h = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    h = h[np.isfinite(h.view(np.float16))]
    table = {}
    out = getattr(ek, target)(_Factory(ek.Float16, table, 0x7c0000000000).copy(h.view(np.float16)))
    prog = ek.debug_program()
    body = _names(prog, prog["sweeps"][0]["body"])
    assert "CVT_F16_F32" in body
    got = _run(prog, oracle, table, "assembled").vars[out.index]
    f = h.view(np.float16).astype(np.float32)
    if target == "Float64":
        want = f.astype(np.float64)
    elif target == "UInt32":          # Float32 -> UInt32 of DESIGN.md 4: negative values wrap like int32
        want = np.trunc(f).astype(np.int64).astype(np.uint32)
    else:
        want = np.trunc(f).astype(np.int64).astype(np.int32).astype(getattr(np, target.lower()))
    assert (got.view(want.dtype) == want).all()


def _rejects(ek, build, what):
    r = build()
    with pytest.raises(ek.EnokiError) as e:
        ek.debug_plan()
    assert "Float16" in str(e.value), (what, str(e.value))
    del r


@pytest.mark.parametrize("what", ["add", "mul", "neg", "sqrt", "lt", "eq", "fmadd", "mul_nz", "fma_nz", "hsum", "hmax",
                                  "scatter_add", "floor"])
def test_arithmetic_comparisons_and_reductions_are_rejected(ek, what):
    table = {}
    F = _Factory(ek.Float16, table, 0x7c0000000000)
    a, b = F.copy(np.ones(4096, np.float16)), F.copy(np.ones(4096, np.float16))
    idx = _Factory(ek.UInt32, table, 0x7a0000000000).copy(np.zeros(4096, np.uint32))
    build = {
        "add": lambda: a + b, "mul": lambda: a * b, "neg": lambda: -a, "sqrt": lambda: ek.sqrt(a),
        "lt": lambda: a < b, "eq": lambda: ek.eq(a, b), "fmadd": lambda: ek.fmadd(a, b, a),
        "mul_nz": lambda: ek.mul_nz(a, b), "fma_nz": lambda: ek.fma_nz(a, b, a), "hsum": lambda: ek.hsum(a),
        "hmax": lambda: ek.hmax(a), "floor": lambda: ek.floor(a),
        "scatter_add": lambda: ek.scatter_add(a, b, idx),
    }[what]
    _rejects(ek, build, what)


def test_the_tape_refuses_float16(ek):
    L = ek.lib()
    assert L.ek_tape_append_leaf(ek.EK_FLOAT16, 16) == 0
    assert "Float16" in L.ek_last_error().decode()


def test_whos_names_the_type_f16(ek):
    table = {}
    a = _Factory(ek.Float16, table, 0x7c0000000000).copy(np.ones(8, np.float16))
    assert any(" f16 " in line and line.split()[0] == str(a.index) for line in ek.cuda_whos().splitlines())
