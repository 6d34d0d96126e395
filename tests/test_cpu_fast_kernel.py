"""CPU: the 32-bit fast sweep kernel ITSELF (enoki_b200/csrc/ek_sweep_fast.cu compiled as host code, tests/cpu_kernel)
executes the lowered programs of the emulator test cases -- random expression DAGs, histograms (privatised bins), group
splitting, reductions, overlapping scatters -- and has to reproduce the expected values.  The numpy interpreter
(ek_emulator.py) still runs the sweeps the fast kernel does not take (size-1 groups, 64-bit programs)."""
import numpy as np
import pytest

import test_cpu_emulator as base
from fast_kernel_emu import FastKernelEmulator


@pytest.fixture(autouse=True)
def native_kernel(monkeypatch):
    monkeypatch.setattr(base, "Emulator", FastKernelEmulator)
    yield


@pytest.mark.parametrize("seed", range(0, 150, 5))
def test_random_dags_on_the_host_compiled_kernel(ek, oracle, P, seed):
    import gc
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()
    # (sizes 1 and 33 give size-1 / tiny groups: those seeds would not reach the kernel -> pick seeds whose n is wide)
    rng = np.random.default_rng(5000 + seed)
    n = int(rng.choice([1, 33, 1000, 4097]))
    if n < 1000:
        pytest.skip("size-1 / 33-element case: not a fast-kernel sweep")
    before = FastKernelEmulator.native_sweeps
    skip = base._case(ek, oracle, P, seed)
    gc.collect()
    if skip:
        pytest.skip(skip)
    if FastKernelEmulator.native_sweeps == before:
        pytest.skip("this DAG uses an operation outside the fast kernel's set: every sweep took the general form")


@pytest.mark.parametrize("n_bins,n", [(31, 5000), (31, 40_003), (300, 9000), (2000, 9000)])
def test_histogram_on_the_host_compiled_kernel(ek, oracle, P, n_bins, n):
    import gc
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()
    base._case_histogram(ek, oracle, P, n_bins, n)
    gc.collect()


def test_group_splitting_on_the_host_compiled_kernel(ek, oracle, P):
    import gc
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()
    assert base._case_many_outputs(ek, oracle, P) >= 2
    gc.collect()


def test_side_effect_order_on_the_host_compiled_kernel(ek, oracle, P):
    base.test_side_effects_run_in_recording_order(ek, oracle, P)


def _differential(ek, oracle, table, outputs, float_tol=()):
    """Runs the pending trace on the numpy interpreter (assembler's program form) and on the host-compiled fast kernel
    (lowered form) and compares every output bit for bit (`float_tol`: names compared with 1e-5 relative instead)."""
    from ek_emulator import Emulator
    prog = ek.debug_program()
    ref = Emulator(oracle, {k: np.array(v, copy=True) for k, v in table.items()}, base._Factory.addresses)
    ref.run(prog)
    nat = FastKernelEmulator(oracle, {k: np.array(v, copy=True) for k, v in table.items()}, base._Factory.addresses)
    before = FastKernelEmulator.native_sweeps
    nat.run(prog)
    assert FastKernelEmulator.native_sweeps > before
    for name, var in outputs.items():
        a, b = ref.vars[var.index], nat.vars[var.index]
        assert a.shape == b.shape and a.dtype == b.dtype, (name, a.shape, b.shape, a.dtype, b.dtype)
        if name in float_tol:
            scale = np.abs(a[np.isfinite(a)].astype(np.float64)).sum() if a.size == 1 or name.startswith("sum") else max(float(np.abs(a[np.isfinite(a)]).max()), 1e-30)
            assert np.allclose(a.astype(np.float64), b.astype(np.float64), rtol=0, atol=1e-5 * max(scale, 1e-30), equal_nan=True), name
        else:
            av, bv = a.view(np.uint8), b.view(np.uint8)
            assert (av == bv).all(), (name, a[:8], b[:8], int((av != bv).sum()))
    ek.lib().ek_debug_discard_side_effects()


@pytest.mark.parametrize("n", [4097, 20_011])
def test_directed_programs_numpy_vs_host_compiled_kernel(ek, oracle, P, n):
    """The programs of the sweep-kernel A/B battery (tests/sweep_battery.py `directed`): mask outputs (8-bit stores)
    reused as staged 8-bit inputs, global gather / scatter / scatter_add with out-of-range indices masked off, signed
    integer operations, rounding conversions, literal operands in every position, min / max / product / count
    reductions, the guarded multiply-adds of the tape."""
    import gc
    from enoki_b200 import Float32, UInt32, Int32, Mask, gather, scatter, scatter_add, fmadd, select, hsum, hmin, hmax, hprod
    import enoki_b200 as E
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()
    rng = np.random.default_rng(n)
    table = {}
    F = base._Factory(Float32, table, 0x7f0000000000); U = base._Factory(UInt32, table, 0x7a0000000000)
    xs_n = [rng.uniform(-4, 4, n).astype(np.float32) for _ in range(4)]
    xs_n[0][:5] = [0.0, -0.0, np.inf, np.nan, 1e-41]
    x0, x1, x2, x3 = (F.copy(a) for a in xs_n)

    # -- masks as outputs, then as staged inputs of a second evaluation
    m1 = x0 > x1; m2 = x2 <= 0.5
    m = (m1 & m2) | ~m1
    _differential(ek, oracle, table, {"mask": m})
    # (give the mask storage so that the next trace stages it as bytes)
    m_n = ((xs_n[0] > xs_n[1]) & (xs_n[2] <= 0.5)) | ~(xs_n[0] > xs_n[1])
    M = base._Factory(Mask, table, 0x7b0000000000).copy(m_n)
    sel = select(M, x0, x1 * 2.0)
    cnt = E._reduce("COUNT", M, UInt32)
    _differential(ek, oracle, table, {"select": sel, "count": cnt})
    del sel, cnt, m, m1, m2

    # -- global gather / scatter_add (6000-entry targets: beyond the shared-memory paths), masked out-of-range indices
    mm = 6000
    src_n = rng.uniform(-1, 1, mm).astype(np.float32)
    idx_n = rng.integers(0, mm + 50, n).astype(np.uint32)
    S = F.copy(src_n); IDX = U.copy(idx_n); TU = U.copy(np.zeros(mm, np.uint32)); TF = F.copy(np.zeros(mm, np.float32))
    ok = IDX < UInt32(mm)
    g = gather(Float32, S, IDX, ok) * x1
    scatter_add(TU, IDX & UInt32(7), IDX, ok)
    scatter_add(TF, x2, IDX, ok)
    _differential(ek, oracle, table, {"gather": g, "add_u32": TU, "add_f32": TF}, float_tol=("add_f32",))
    del g, ok

    # -- index arithmetic with literals, signed operations, conversions
    i = UInt32.arange(n)
    h = i * np.uint32(2654435761) + np.uint32(974711)
    h = (h ^ (h >> 15)) * np.uint32(2246822519)
    s = Int32(x0 * 1000.0)
    s2 = E.max_(s >> Int32(3), -abs(s))
    tof = Float32(s) + Float32(h)
    lt = s < Int32(0)
    _differential(ek, oracle, table, {"hash": h, "signed": s2, "tofloat": tof, "lt": lt})
    del h, s, s2, tof, lt, i

    # -- literal operands in every position
    a = fmadd(x0, 1.5, x1); b = fmadd(x0, x1, -0.75); c = 2.0 - x2; d = 3.0 / x3
    e_ = select(x0 >= 0.25, Float32(1.5), x1); f_ = E.min_(abs(x1), 2.5)
    _differential(ek, oracle, table, {"fma_ub": a, "fma_uc": b, "rsub": c, "rdiv": d, "sel_lit": e_, "min_lit": f_})
    del a, b, c, d, e_, f_

    # -- reductions (NaN-free data) and the guarded multiply-adds
    y0 = F.copy(rng.uniform(-4, 4, n).astype(np.float32)); y1 = F.copy(rng.uniform(-4, 4, n).astype(np.float32))
    r_min = hmin(y0 * y1); r_max = hmax(E.sin(y1)); r_sum = hsum(y0 * y0)
    _differential(ek, oracle, table, {"hmin": r_min, "hmax": r_max, "sum": r_sum}, float_tol=("sum",))
    gc.collect()


@pytest.mark.parametrize("n", [4097, 33_333])
def test_remaining_operations_numpy_vs_host_compiled_kernel(ek, oracle, P, n):
    """Every operation of the fast kernel's set that the other cases do not reach: rounding modes, rcp / rsqrt / log / cos,
    division, the tape's zero-guarded multiply-adds, integer multiply-add, signed min / max / shifts by an array, NOT, all
    comparison flavours with array and literal operands, product / count reductions, and -- with ten input arrays -- the
    direct global loads that take over when the inputs exceed the TMA staging budget."""
    import gc
    from enoki_b200 import Float32, UInt32, Int32, fmadd, select, hsum, hprod
    import enoki_b200 as E
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()
    rng = np.random.default_rng(77 + n)
    table = {}
    F = base._Factory(Float32, table, 0x7f0000000000); U = base._Factory(UInt32, table, 0x7a0000000000)
    xs = [F.copy(rng.uniform(-4, 4, n).astype(np.float32)) for _ in range(4)]
    x0, x1, x2, x3 = xs
    us = [U.copy(rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)) for _ in range(2)]
    u0, u1 = us

    a = E.round_(x0 * 3.3) + E.trunc(x1 * 2.7) + E.ceil(x2) - E.floor(x3)
    b = (E.rcp(x0) + E.rsqrt(abs(x1) + 0.5) + E.log(abs(x2) + 1e-3) * E.cos(x3)) / x1      # (numerator first: DIV, not the reversed form)
    c = E.mul_nz(E.floor(x2) * 0.5, x3)
    _differential(ek, oracle, table, {"round": a, "rcp_log_cos_div": b, "nz": c})
    del a, b, c

    s = Int32(x0 * 1000.0); t = Int32(x1 * 1000.0)
    sh = U.copy(rng.integers(0, 32, n).astype(np.uint32)); sh7 = base._Factory(Int32, table, 0x7c0000000000).copy(rng.integers(0, 8, n).astype(np.int32))
    d = fmadd(u0, sh, u1)                                   # integer multiply-add
    e_ = E.min_(Int32(100) - t, s) + E.max_(s * Int32(3), t)
    g = ((u0 ^ u1) << sh) ^ UInt32((s * Int32(5)) >> sh7)
    h = ~u1
    _differential(ek, oracle, table, {"mad": d, "minmax": e_, "shifts": g, "not": h})
    del d, e_, g, h

    m = (u0.neq_(u1) | (s >= Int32(5))) ^ ((x0 <= x1) & x2.neq_(x3)) ^ (u0 > UInt32(0x80000000)) ^ (s <= t) ^ u0.eq_(UInt32(7)) ^ (x2 >= x3)
    sel = select(E.floor(x0).eq_(E.floor(x1)), x2, x3)
    _differential(ek, oracle, table, {"cmp": m, "sel": sel})
    del m, sel, s, t, sh, sh7

    y = F.copy(rng.uniform(0.999, 1.001, n).astype(np.float32))
    mk = x0 > 0.5
    prod = hprod(y); cnt = E._reduce("COUNT", mk, UInt32); tot = hsum(UInt32(u0 >> UInt32(12)))
    # (the numpy interpreter folds the product in float64, the kernel in a float32 tree: ~sqrt(n) eps apart)
    prog = ek.debug_program()
    _differential(ek, oracle, table, {"count": cnt, "usum": tot})
    from ek_emulator import Emulator
    nat = FastKernelEmulator(oracle, {k: np.array(v, copy=True) for k, v in table.items()}, base._Factory.addresses)
    nat.run(prog)
    want = float(np.prod(table[y.index].astype(np.float64)))
    assert abs(float(nat.vars[prod.index][0]) - want) <= 1e-3 * abs(want)
    del prod, cnt, tot, mk, y

    # ten wide inputs in one expression: beyond the staging budget (8 slot units) -> FOP_LDG_32
    many = [F.copy(rng.uniform(-1, 1, n).astype(np.float32)) for _ in range(10)]
    acc = many[0]
    for k in range(1, 10):
        acc = fmadd(acc, many[k], many[(k * 3) % 10]) if k % 2 else acc * many[k] + x0
    prog = ek.debug_program()
    assert any("LDG_32" in [prog["fops"][t[0]] for t in sw["fast"]["body"]] for sw in prog["sweeps"] if "fast" in sw), "no direct global load in the lowered program"
    _differential(ek, oracle, table, {"ldg": acc})
    gc.collect()


# device operation -> a wide 32-bit program that needs it; none of these has a fast-kernel form
_GENERAL_ONLY = {
    "DIV_I32": lambda E, a: a(E.Int32) // a(E.Int32),
    "DIV_U32": lambda E, a: a(E.UInt32) // a(E.UInt32),
    "MOD_I32": lambda E, a: a(E.Int32) % a(E.Int32),
    "MOD_U32": lambda E, a: a(E.UInt32) % a(E.UInt32),
    "MULHI_I32": lambda E, a: E.mulhi(a(E.Int32), a(E.Int32)),
    "MULHI_U32": lambda E, a: E.mulhi(a(E.UInt32), a(E.UInt32)),
    "POPC_32": lambda E, a: E.popcnt(a(E.UInt32)),
    "CLZ_32": lambda E, a: E.lzcnt(a(E.UInt32)),
    "CTZ_32": lambda E, a: E.tzcnt(a(E.UInt32)),
    "SEXT8": lambda E, a: a(E.Int8) + a(E.Int8),                   # (8-bit staged loads and stores do have a form)
    "ZEXT8": lambda E, a: a(E.UInt8) + a(E.UInt8),
    "LD_U16": lambda E, a: E.UInt32(a(E.UInt16)) + 1,
    "ST_16": lambda E, a: E.UInt16(a(E.UInt8)),
    "GATHER_U8": lambda E, a: E.gather(E.UInt8, a(E.UInt8), a(E.UInt32)),
    "SCATTER_8": lambda E, a: E.scatter(a(E.UInt8), E.UInt8(3), a(E.UInt32)),
    "SCATTER_16": lambda E, a: E.scatter(a(E.UInt16), E.UInt16(3), a(E.UInt32)),
}


def _c2(E, a):
    x0, x1, x2, x3 = (a(E.Float32) for _ in range(4))
    t = E.fmadd(x0, x1, x2)
    return E.fmadd(E.sin(E.fmadd(x3, E.exp(-(t * t)), x0)), x1, E.sqrt(abs(t)))


def _c3(E, a):
    tab, bins, hist = a(E.Float32, 31), a(E.UInt32, 31), a(E.Float32, 31)
    idx = E.UInt32((a(E.Float32) + 4.0) * 31.0 / 8.0)
    mask = idx < E.UInt32(31)
    w = E.gather(E.Float32, tab, idx, mask)
    E.scatter_add(bins, E.UInt32(1), idx, mask)
    E.scatter_add(hist, w, idx, mask)


@pytest.mark.parametrize("case", [*_GENERAL_ONLY, "C2", "C3", "C2_fast_mode_off"])
def test_which_programs_the_fast_kernel_runs(ek, case):
    """The fast kernel's operation set is what lower_fast can lower (fop_of in ek_eval.cpp): a wide 32-bit program that
    uses one operation outside it runs on the general kernel as a whole, so its sweep in ek_debug_program() has no "fast"
    section.  C2 and C3 lower, unless ek_set_fast_mode(0) has switched the fast kernel off."""
    import gc
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()
    n = 5000                                        # wide: n > 4096
    mapped = []

    def a(cls, size=n):                             # a mapped array (the program is planned, never run)
        mapped.append(cls.map(0x770000000000 +0x1000000 * len(mapped), size))
        return mapped[-1]
    build = _GENERAL_ONLY.get(case) or (_c3 if case == "C3" else _c2)
    L = ek.lib()
    old = L.ek_fast_mode()
    try:
        L.ek_set_fast_mode(0 if case == "C2_fast_mode_off" else 1)
        out = build(ek, a)
        prog = ek.debug_program()
    finally:
        L.ek_set_fast_mode(old)
    sweeps = [sw for sw in prog["sweeps"] if sw["n"] == n]
    assert len(sweeps) == 1
    sw = sweeps[0]
    if case in _GENERAL_ONLY:
        ops = {prog["ops"][t[0]] for sec in ("init", "body", "fini") for t in sw[sec]}
        assert case in ops, ops
        assert "fast" not in sw
    else:
        assert ("fast" in sw) == (case != "C2_fast_mode_off")
    del out, mapped
    L.ek_debug_discard_side_effects()


def test_block_size_128_instantiation():
    """The same cases once more with the fast kernel restricted to its 128-thread instantiation (EK_FAST_T=128 is read once
    per process, hence the child process): operand offsets, group strides and the reduction epilogue for T = 128."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, EK_FAST_T="128")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(root, "tests", "test_cpu_fast_kernel.py"), "-q", "-x",
                        "-k", "not block_size_128", "-p", "no:cacheprovider"], capture_output=True, text=True, timeout=1200, env=env, cwd=root)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout
