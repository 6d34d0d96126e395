"""CPU: the reduction programs of tests/test_gpu_horizontal.py through the planner, the assembler and the numpy
interpreter of the sweep ISA (tests/ek_emulator.py) over fake device addresses.  Only checks that do not depend on the
fold order are kept (integers, and floats on integer-valued data), so this runs the reduction identities, the class
chosen for narrow types, fused and standalone RACC, the mask normalisation of count / any / all and the group split
above EK_MAX_RED reductions without a GPU.  psum, compress, fill and reverse are not sweep programs and stay GPU-only."""
import gc

import numpy as np
import pytest

from ek_emulator import Emulator
import test_gpu_horizontal as hz


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
    """put(cls, array, poison) for the builders: maps a fake device address and hands the data to the emulator."""
    def __init__(self):
        self.table, self.base = {}, 0x700000000000

    def __call__(self, cls, arr, poison):
        address = self.base + 0x10000000 * (len(self.table) + 1)
        r = cls.map(address, len(arr))
        self.table[r.index] = np.ascontiguousarray(arr)
        return r


def _run(ek, oracle, build):
    """Record the cases, execute every planned sweep on the emulator, and compare each result exactly."""
    put = _Put()
    cases = build(put)
    prog = ek.debug_program()
    emu = Emulator(oracle, put.table)
    emu.run(prog)
    bad = []
    for label, var, want in cases:
        assert var.index in emu.vars, f"{label}: result was not produced by any sweep"
        want = np.asarray(want)
        got = np.ascontiguousarray(emu.vars[var.index]).reshape(-1)
        if want.dtype.kind == "f":
            ok = got.dtype == want.dtype and got[0] == want
        elif got.dtype == np.bool_ or want.dtype == np.uint8 and label.startswith(("any", "all")):
            ok = int(got.view(np.uint8)[0] if got.dtype == np.bool_ else got[0]) == int(want)
        else:                                  # (narrow results sit in the low bytes of the 32-bit result word)
            ok = (got.view(np.uint8)[:want.dtype.itemsize] == want.reshape(1).view(np.uint8)).all()
        if not ok:
            bad.append(f"{label}: got {got[:1]!r}, want {want!r}")
    assert not bad, "; ".join(bad)
    return prog, emu


@pytest.mark.parametrize("n", [2, 31, 1025, 4097])
@pytest.mark.parametrize("tname", hz.TYPES32 + hz.TYPES64)
def test_reductions_on_the_emulator(ek, oracle, clean, tname, n):
    _run(ek, oracle, lambda put: hz.reduction_cases(ek, put, tname, n, seed=n))


@pytest.mark.parametrize("n", [2, 31, 4097])
def test_mask_reductions_on_the_emulator(ek, oracle, clean, n):
    _run(ek, oracle, lambda put: hz.mask_cases(ek, put, n, seed=n))


def test_many_classes_in_one_sweep_on_the_emulator(ek, oracle, clean):
    prog, _ = _run(ek, oracle, lambda put: hz.mixed_class_cases(ek, put, 4097, seed=1))
    assert len(prog["sweeps"]) == 1


@pytest.mark.parametrize("n", [31, 4097])
def test_more_reductions_than_one_kernel_holds_on_the_emulator(ek, oracle, clean, n):
    """40 reductions > EK_MAX_RED: the planner splits the group instead of failing, and every result is right."""
    prog, _ = _run(ek, oracle, lambda put: hz.many_reductions(ek, put, n, seed=n))
    assert len(prog["sweeps"]) >= 2
    assert all(sum(1 for i in sw["fini"] if prog["ops"][i[0]] == "RFIN") <= 32 for sw in prog["sweeps"])
