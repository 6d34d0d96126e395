"""CPU: the conversion matrix and the 64-bit operation cases of tests/test_gpu_conversions.py through the planner, the
assembler and the numpy interpreter of the sweep ISA (tests/ek_emulator.py), in both program forms; the golden
conversions of the reference against exact Python where they are defined; Float32 -> UInt32 on the fast kernel's own
source compiled for the host (tests/cpu_kernel)."""
import gc

import numpy as np
import pytest

from ek_emulator import Emulator
from fast_kernel_emu import FastKernelEmulator
from test_cpu_gather_scatter import _Put
import test_gpu_conversions as cv
import test_gpu_gather_scatter as gs


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


def _run(ek, oracle, build, emulator=Emulator):
    put = _Put()
    case = build(put)
    gs.check_plan(ek, cv.case_plan(case))
    prog = ek.debug_program()
    emu = emulator(oracle, put.table, put.addresses)
    emu.run(prog)

    def got(var):
        assert var.index in emu.vars, "result was not produced by any sweep"
        a = emu.vars[var.index]
        return a.view(np.uint8) if a.dtype == np.bool_ else a
    case.verify(got)
    del case
    ek.lib().ek_debug_discard_side_effects()
    return prog


@pytest.mark.parametrize("n", [1, 4097])
@pytest.mark.parametrize("src,group", sorted({(s, g) for s, g, _ in cv.CONVERT_PARAMS}))
def test_conversion_matrix_on_the_emulator(ek, oracle, clean, src, group, n):
    dsts = dict(cv.groups(src))[group]
    _run(ek, oracle, lambda put: cv.convert_case(ek, put, src, dsts, n, seed=n + cv.TYPES.index(src)))


@pytest.mark.parametrize("form", ["array", "literal", "scalar"])
@pytest.mark.parametrize("tname", cv.WIDE)
def test_ops64_on_the_emulator(ek, oracle, clean, program_form, tname, form):
    if program_form == "lowered":
        pytest.skip("64-bit programs have no lowered form")
    ops = cv.ops64(tname, form)
    for n in (1, 4097):
        for k in range(0, len(ops), 8):
            _run(ek, oracle, lambda put: cv.ops_case(ek, put, tname, ops[k:k + 8], n, form, seed=n + k))


def test_float_to_uint32_on_the_host_compiled_kernel(ek, oracle, clean, program_form):
    """Float32 -> UInt32 / Int32 / narrow types and floor2int / ceil2int on 2^20 + 7 elements whose threads are all in
    range, all out of range or mixed, on the fast kernel's source compiled for the host."""
    if program_form == "lowered":
        pytest.skip("the host-compiled kernel always runs the lowered form")
    before = FastKernelEmulator.native_sweeps
    prog = _run(ek, oracle, lambda put: cv.convert_case(ek, put, "Float32", dict(cv.groups("Float32"))["32"],
                                                         (1 << 20) + 7, seed=3), emulator=FastKernelEmulator)
    assert all("fast" in sw for sw in prog["sweeps"])
    assert FastKernelEmulator.native_sweeps > before


def test_golden_conversions_are_exact_where_defined(program_form):
    """The reference's conversions in convert.npz agree with exact Python wherever the rounded value fits the
    destination, and differ from correct rounding only where its UInt32 -> Float32 rounds twice; the issue-prone rows
    are what the reference computes."""
    if program_form == "lowered":
        pytest.skip("no program involved")
    g = cv.golden()
    for src in cv.TYPES:
        x = g[f"x_{src}"]
        for dst in cv.TYPES:
            for mode in cv.modes_of(src, dst):
                ref = g[f"{src}_{dst}_{mode}"]
                want, defined = cv.exact(src, dst, mode, x)
                ok = (cv.bits(ref) == cv.bits(want)) | ~defined
                if want.dtype.kind == "f":
                    ok |= np.isnan(ref) & np.isnan(want)
                if (src, dst) == ("UInt32", "Float32"):
                    assert (~ok == cv.double_rounded_u32(x)).all()
                    assert (~ok).any(), "no input exercises the reference's double rounding"
                else:
                    assert ok.all(), (src, dst, mode, x[~ok][:4], ref[~ok][:4], want[~ok][:4])
    x = g["x_Float32"]
    at = lambda v: int(np.flatnonzero(np.isnan(x) if np.isnan(v) else x == np.float32(v))[0])
    assert g["Float32_UInt64_0"][at(1e19)] == 0x8ac7230000000000
    assert g["Float32_UInt32_0"][at(np.nan)] == 0x80000000
    assert g["Float32_UInt32_0"][at(5e9)] == 0
    assert g["Float32_UInt32_0"][at(-3e9)] == 0x80000000
    assert g["Float32_UInt32_1"][at(-2.5)] == 0xfffffffd
    assert g["Float32_UInt32_2"][at(-0.7)] == 0
    xd = g["x_Float64"]
    assert g["Float64_UInt64_0"][int(np.flatnonzero(xd == 1e19)[0])] == 0x8ac7230489e80000
