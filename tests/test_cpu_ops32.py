"""CPU: the 32-bit and narrow-integer operation cases of tests/test_gpu_ops32.py through the planner, the assembler and
the numpy interpreter of the sweep ISA (tests/ek_emulator.py), in both program forms, and the Float32 / Int32 / UInt32
ones on the fast kernel's own source compiled for the host (tests/cpu_kernel), with the fast kernel's forms asserted
from the lowered bodies; the exact references against the reference CPU path where it is built."""
import ctypes
import gc

import numpy as np
import pytest

from ek_emulator import Emulator
from fast_kernel_emu import FastKernelEmulator
from test_cpu_conversions import _run
import test_gpu_conversions as cv
import test_gpu_ops32 as o32


@pytest.fixture(autouse=True, params=["assembled", "lowered"])
def program_form(request):
    Emulator.prefer_fast = request.param == "lowered"
    yield request.param
    Emulator.prefer_fast = False


@pytest.fixture()
def clean(ek):
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()
    assert ek.debug_plan() == "", "unevaluated variables of an earlier test are still alive"
    yield
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()


PARAMS = [(t, f) for t in o32.TYPES for f in o32.FORMS]


@pytest.mark.parametrize("n", [1, 4097])
@pytest.mark.parametrize("tname,form", PARAMS)
def test_ops32_on_the_emulator(ek, oracle, clean, tname, form, n):
    for k, (ops, keep, _) in enumerate(o32.programs_of(tname, form)):
        build = lambda put: cv.ops_case(ek, put, tname, ops, n, form, seed=n + 31 * k, keep=keep, oracle=oracle)
        _run(ek, oracle, build)


@pytest.mark.parametrize("tname,form", [(t, f) for t in o32.FAST_TYPES + ("Int8", "UInt8") for f in o32.FORMS])
def test_ops32_on_the_host_compiled_kernel(ek, oracle, clean, program_form, tname, form):
    """4097 elements: the programs of the fast kernel's operations run on its host-compiled source and reach every
    form of it that the GPU test asserts; the others have no fast form (8-bit types: their comparisons and selects of
    staged inputs run there, their arithmetic does not)."""
    if program_form == "lowered":
        pytest.skip("the host-compiled kernel always runs the lowered form")
    programs = []
    for k, (ops, keep, on_fast) in enumerate(o32.programs_of(tname, form)):
        before = FastKernelEmulator.native_sweeps
        build = lambda put: cv.ops_case(ek, put, tname, ops, 4097, form, seed=4097 + 31 * k, keep=keep, oracle=oracle)
        prog = _run(ek, oracle, build, emulator=FastKernelEmulator)
        if on_fast:
            assert all(sw["config"]["fast"] for sw in prog["sweeps"] if sw["n"] > 1), ops
            assert FastKernelEmulator.native_sweeps > before
            programs.append(prog)
        else:
            assert not any("fast" in sw for sw in prog["sweeps"]), ops
    if tname in o32.FAST_TYPES:
        o32.check_fast_forms(tname, form, programs)


def test_references_match_the_reference_cpu_path(ref, oracle, program_form):
    """The exact Float32 references of the operation cases equal the reference CPU path bit for bit on their operand
    rows, except min / max where an operand is NaN or the operands are equal (+-0 ties): there the reference returns
    its first operand and this backend its second (DESIGN.md 4)."""
    if program_form == "lowered":
        pytest.skip("no program involved")
    if ref is None:
        pytest.skip("the reference CPU path (oracle/_ref/libenoki_ref.so) is not built")
    a, b, c = cv.float_operands("Float32", 700, np.random.default_rng(1))
    x, y, z = (np.array(v, np.float64).astype(np.float32) for v in (a, b, c))
    n = len(x)
    P = lambda v: v.ctypes.data_as(ctypes.c_void_p)
    bad = []
    for op in o32.REF_UNARY + o32.REF_BINARY + ("fma",):
        got = np.zeros(n, np.float32)
        if op == "fma":
            ref.ref_fmadd_f32(P(x), P(y), P(z), P(got), ctypes.c_size_t(n))
        elif op in o32.REF_BINARY:
            assert ref.ref_binary_f32(op.encode(), P(x), P(y), P(got), ctypes.c_size_t(n)) == 0
        else:
            assert ref.ref_unary_f32(op.encode(), P(x), P(got), ctypes.c_size_t(n)) == 0
        want, _ = cv.expected("Float32", op, a, b if op in o32.REF_BINARY + ("fma",) else None, c if op == "fma" else None,
                              oracle=oracle)
        ok = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
        if op in ("min", "max"):
            div = np.isnan(x) | np.isnan(y) | (x == y)
            assert (~ok <= div).all() and (~ok).any(), op        # they differ there, and only there
            ok |= div
        if not ok.all():
            k = int(np.flatnonzero(~ok)[0])
            bad.append(f"{op}: {int((~ok).sum())} differ, first a={x[k]!r} b={y[k]!r} c={z[k]!r}: ref {got[k]!r}, "
                       f"exact {want[k]!r}")
    assert not bad, "; ".join(bad)
