"""CPU: the 32-bit gather / scatter / scatter_add cases of tests/test_gpu_gather_scatter.py through the planner, the
assembler and the numpy interpreter of the sweep ISA (tests/ek_emulator.py), in both program forms; the lowering each
case must get at every threshold (planning only, at any size); the signed-zero bins on the host-compiled fast kernel
(tests/cpu_kernel); and the rejection of strides that do not fit the program's 15-bit field."""
import gc

import numpy as np
import pytest

from ek_emulator import Emulator
from fast_kernel_emu import FastKernelEmulator
import test_gpu_gather_scatter as gs


@pytest.fixture(autouse=True, params=["assembled", "lowered"])
def program_form(request):
    """Every test runs on the assembler's program and on the program lowered for the 32-bit fast kernel (where the
    sweep has one)."""
    Emulator.prefer_fast = request.param == "lowered"
    yield request.param
    Emulator.prefer_fast = False


@pytest.fixture()
def clean(ek):
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()
    assert ek.debug_plan() == "", "unevaluated variables of an earlier test are still alive"
    yield
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()


class _Put:
    """put(cls, array, guard) for the builders: maps a fake device address and hands the data (without the guard) to
    the emulator, which reaches gather sources and scatter targets by address."""
    def __init__(self):
        self.table, self.addresses, self.base = {}, {}, 0x700000000000

    def __call__(self, cls, arr, guard):
        address = self.base + 0x10000000 * (len(self.table) + 1)
        r = cls.map(address, len(arr))
        self.table[r.index] = np.ascontiguousarray(arr)
        self.addresses[address] = r.index
        return r


def _run(ek, oracle, build, emulator=Emulator):
    put = _Put()
    case = build(put)
    gs.check_plan(ek, case)
    emu = emulator(oracle, put.table, put.addresses)
    emu.run(ek.debug_program())

    def got(var):
        assert var.index in emu.vars, "result was not produced by any sweep"
        a = emu.vars[var.index]
        return a.view(np.uint8) if a.dtype == np.bool_ else a
    case.verify(got)
    ek.lib().ek_debug_discard_side_effects()
    return emu


T32 = ("Float32", "Int32", "UInt32")


@pytest.mark.parametrize("n", [31, 4097])
@pytest.mark.parametrize("itype", ["UInt32", "Int32"])
@pytest.mark.parametrize("tname", T32)
def test_gather_on_the_emulator(ek, oracle, clean, tname, itype, n):
    for size in (1, 31, 4096, 4097):
        _run(ek, oracle, lambda put: gs.gather_case(ek, put, tname, itype, n, size, seed=n + size))


@pytest.mark.parametrize("n", [1, 31, 4097])
@pytest.mark.parametrize("tname", T32)
def test_scatter_on_the_emulator(ek, oracle, clean, tname, n):
    for part in "AB":
        _run(ek, oracle, lambda put: gs.scatter_case(ek, put, tname, n, seed=n, part=part))


@pytest.mark.parametrize("count", gs.BIN_COUNTS)
@pytest.mark.parametrize("tname", T32)
def test_scatter_add_on_the_emulator(ek, oracle, clean, tname, count):
    _run(ek, oracle, lambda put: gs.scatter_add_case(ek, put, tname, count, 4097, seed=count))
    _run(ek, oracle, lambda put: gs.scatter_add_case(ek, put, tname, count, 4097, seed=count + 1, heavy=True))


@pytest.mark.parametrize("count", [31, 32, 33, 129, 1024, 1025, 50_000])
def test_signed_zero_on_the_emulator(ek, oracle, clean, count):
    _run(ek, oracle, lambda put: gs.signed_zero_case(ek, put, count, 4097, seed=count)[0])


@pytest.mark.parametrize("kind", ["equal", "above", "below", "shared", "signed"])
def test_implied_mask_on_the_emulator(ek, oracle, clean, kind):
    _run(ek, oracle, lambda put: gs.implied_case(ek, put, kind, 4097, seed=3))


def _plan_only(ek, build):
    put = _Put()
    case = build(put)
    ops = gs.check_plan(ek, case)
    del case
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()
    return ops


@pytest.mark.parametrize("n", [2, 4096, 4097, gs.BIG])
def test_lowering_at_every_threshold(ek, clean, program_form, n):
    """Which lowering each size gets: tables of <= 4096 words in shared memory, 4097 global; bins of <= 1024 words
    privatised, 1025 global; signed or 64-bit indices never take the shared-memory forms; size-1 sweeps never do."""
    if program_form == "lowered":
        pytest.skip("planning only: one program form is enough")
    E = ek
    for size, want in ((4096, "GATHER_32_SMEM"), (4097, "GATHER_32")):
        for itype, w in (("UInt32", want), ("Int32", "GATHER_32"), ("UInt64", "GATHER_32")):
            def build(put, size=size, itype=itype, w=w):
                c = gs.Case()
                S = E.Float32.map(0x710000000000, size)
                X = getattr(E, itype).map(0x720000000000, n)
                c.keep += [S, E.gather(E.Float32, S, X, X < getattr(E, itype)(7))]
                c.plan.append(w)
                if w == "GATHER_32_SMEM":
                    c.absent.append("GATHER_32")
                return c
            _plan_only(ek, build)
    for tname in ("Float32", "Int32", "UInt32"):
        for count in gs.BIN_COUNTS:
            for itype in ("UInt32", "Int32"):
                def build(put, tname=tname, count=count, itype=itype):
                    c = gs.Case()
                    Tg = getattr(E, tname).map(0x730000000000, count)
                    X = getattr(E, itype).map(0x740000000000, n)
                    E.scatter_add(Tg, getattr(E, tname)(1), X)
                    c.keep.append(Tg)
                    c.plan.append(gs.add_lowering(tname, count, n, itype))
                    return c
                _plan_only(ek, build)


def test_smem_zero_marks_float_bins(ek, clean, program_form):
    """SMEM_ZERO carries dst = 1 for float bins (filled with -0.0) and 0 for integer bins, in both program forms."""
    E = ek
    Tf = E.Float32.map(0x750000000000, 31)
    Ti = E.UInt32.map(0x760000000000, 31)
    X = E.UInt32.map(0x770000000000, 5000)
    E.scatter_add(Tf, E.Float32(1.0), X)
    E.scatter_add(Ti, E.UInt32(1), X)
    prog = ek.debug_program()
    sw = [s for s in prog["sweeps"] if s["n"] == 5000][0]
    zero = prog["ops"].index("SMEM_ZERO")
    flags = [ins[2] for ins in sw["init"] if ins[0] == zero]
    assert sorted(flags) == [0, 1]
    if "fast" in sw:
        fzero = prog["fops"].index("SMEM_ZERO")
        assert sorted(t[4] for t in sw["fast"]["init"] if t[0] == fzero) == [0, 1]
    del Tf, Ti, X


def test_signed_zero_on_the_host_compiled_kernel(ek, oracle, clean, program_form):
    """31 float bins (one private copy per thread, then the shuffle-tree flush) on the fast kernel's own source compiled
    for the host, against the IEEE sum of every element."""
    if program_form == "lowered":
        pytest.skip("the host-compiled kernel always runs the lowered form")
    n = 9 * 4096 + 1000
    before = FastKernelEmulator.native_sweeps
    _run(ek, oracle, lambda put: gs.signed_zero_case(ek, put, 31, n, seed=31)[0], emulator=FastKernelEmulator)
    assert FastKernelEmulator.native_sweeps > before


def test_stride_rejection(ek, clean, program_form):
    gs.stride_rejection(ek, 0x7e0000000000)          # (nothing is evaluated: a fake address will do on the host)
    gc.collect()
