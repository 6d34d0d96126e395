"""CPU: the launch paths of tests/test_gpu_launch_paths.py chosen by the planner, checked without a GPU.

The same builders run on fake device addresses; only the path the host selects is asserted: program lengths around
the inline (448) and shared-memory (24 KB) limits of program delivery, literal pools around 128 words, direct loads
beyond the staging budget, scalar and slot splits, and the configuration choose_config picks for every row of the
configuration table (the dry run reports it).  A change to one of these thresholds fails a test here.  Where the numpy
interpreter of the sweep ISA (tests/ek_emulator.py) runs every operation of a case, the values are checked too."""
import gc

import numpy as np
import pytest

from ek_emulator import Emulator, Unsupported
import test_gpu_launch_paths as lp


class Fake:
    """put(cls, array, misaligned): a fake device mapping whose data the emulator reads."""
    def __init__(self):
        self.table, self.k = {}, 0

    def __call__(self, cls, arr, misaligned=False):
        self.k += 1
        r = cls.map(0x700000000000 + 0x10000000 * self.k + (arr.itemsize if misaligned else 0), len(arr))
        self.table[r.index] = np.ascontiguousarray(arr)
        return r


@pytest.fixture()
def clean(ek):
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()
    assert ek.debug_plan() == "", "unevaluated variables of an earlier test are still alive"
    yield ek
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()


def emulate(ek, oracle, put, cases, prog):
    """Run the planned sweeps on the emulator and compare every case exactly; False when it lacks an operation."""
    emu = Emulator(oracle, put.table)
    try:
        emu.run(prog)
    except Unsupported:
        return False
    for label, var, want in cases:
        assert var.index in emu.vars, f"{label}: not produced by any sweep"
        got = np.ascontiguousarray(emu.vars[var.index]).reshape(-1)
        want = np.asarray(want)
        got = got.view(want.dtype) if got.dtype.itemsize == want.dtype.itemsize else got.astype(want.dtype)
        assert lp.same_bits(got, want), label
    return True


@pytest.mark.parametrize("target", [lp.INLINE_PROG, lp.INLINE_PROG + 1, lp.SMEM_PROG, lp.SMEM_PROG + 1, 4000])
@pytest.mark.parametrize("tname", ["Float64", "Float32"])
def test_program_delivery_plan(clean, oracle, tname, target):
    ek = clean
    put = Fake()
    cases, prog = lp.tuned(ek, lambda L: lp.delivery_case(ek, put, 5000, L, tname), target,
                           lambda p: lp.prog_len(p["sweeps"][0]) if len(p["sweeps"]) == 1 else None, target - 4)
    sw = prog["sweeps"][0]
    assert sw["init"] and sw["fini"]
    cfg = sw["config"]
    assert cfg["prog_in_smem"] == (target <= lp.SMEM_PROG)
    assert cfg["inline_prog"] == (target <= lp.INLINE_PROG)
    assert cfg["fast"] == 0 or tname == "Float32"
    if target <= lp.SMEM_PROG + 1:
        assert emulate(ek, oracle, put, cases[:1], prog)


@pytest.mark.parametrize("target", [lp.INLINE_PROG, lp.INLINE_PROG + 1])
def test_fast_kernel_program_length_plan(clean, target):
    ek = clean
    cases, prog = lp.fast_tuned(ek, Fake(), 3 * 4096 + 5, target)
    assert prog["sweeps"][0]["config"]["fast"] == (1 if target == lp.INLINE_PROG else 0)


@pytest.mark.parametrize("words", [lp.LIT_INLINE - 1, lp.LIT_INLINE, lp.LIT_INLINE + 1, lp.LIT_INLINE + 2, 3300])
def test_literal_pool_plan(clean, oracle, words):
    ek = clean
    put = Fake()
    cases, prog = lp.tuned(ek, lambda k: lp.literal_case(ek, put, 5000, k), words,
                           lambda p: len(p["sweeps"][0]["lits"]), words)
    sw = prog["sweeps"][0]
    assert (sw["config"]["fast"] == 1) == (words <= lp.LIT_INLINE + 2)
    assert sw["config"]["inline_lit"] == (words <= lp.LIT_INLINE)
    if words == 3300:
        assert sw["config"]["ctas_per_sm"] < 4
    assert emulate(ek, oracle, put, cases, prog)


def test_literal_pair_and_pool_overflow_plan(clean):
    ek = clean
    cases = lp.straddle_case(ek, Fake(), 5000)
    sw = [s for s in ek.debug_program()["sweeps"] if len(s["lits"]) == lp.LIT_INLINE + 1]
    assert len(sw) == 1
    del cases
    gc.collect()
    put = Fake()
    cases = lp.literal_case(ek, put, 5000, 2200) + lp.literal_case(ek, put, 5000, 2200, base=5000)
    assert [len(s["lits"]) for s in ek.debug_program()["sweeps"]] == [2200, 2200]
    del cases
    gc.collect()
    cases = lp.literal_case(ek, Fake(), 5000, 4200)
    with pytest.raises(ek.EnokiError, match="uniform pool overflow"):
        ek.debug_program()


def test_direct_load_plan(clean, oracle):
    ek = clean
    put = Fake()
    cases = lp.direct_f32_case(ek, put, 5000)
    prog = ek.debug_program()
    sw = prog["sweeps"][0]
    assert lp.ops(prog, sw).count("LDG_32") == 17 - lp.STAGE_UNITS and len(sw["staged"]) == lp.STAGE_UNITS
    assert "fast" in sw and "LDG_32" in [prog["fops"][i[0]] for i in sw["fast"]["body"]]
    assert emulate(ek, oracle, put, cases, prog)
    del cases
    gc.collect()
    cases = lp.direct_f64_case(ek, put, 5000)
    prog = ek.debug_program()
    sw = prog["sweeps"][0]
    assert lp.ops(prog, sw).count("LDG_64") == 1 and len(sw["staged"]) == lp.STAGE_UNITS // 2
    del cases
    gc.collect()
    cases = lp.direct_narrow_case(ek, put, 5000)
    prog = ek.debug_program()
    sw = prog["sweeps"][0]
    o = lp.ops(prog, sw)
    assert len(sw["staged"]) == lp.STAGE_UNITS
    assert [o.count(k) for k in ("LDG_S8", "LDG_U8", "LDG_S16", "LDG_U16", "LDG_64")] == [1, 2, 1, 1, 2]


def test_misaligned_staged_plan(clean):
    ek = clean
    cases = lp.staged_mixed_case(ek, Fake(), 5000)
    prog = ek.debug_program()
    sw = prog["sweeps"][0]
    assert sorted(es for _v, _u, es in sw["staged"]) == [1, 2, 2, 8]
    assert {"LD_S8", "LD_S16", "LD_U16", "LD_64"} <= set(lp.ops(prog, sw))


@pytest.mark.parametrize("row", lp.CONFIG_ROWS, ids=lambda r: "V%d_T%d_s%d_c%d" % r[3])
def test_configuration_table(clean, row):
    """Every row lands on its candidate: as the launcher picks it, and as the test's own model of choose_config does."""
    ek = clean
    with lp.fast_mode(ek, False):
        cases = lp.config_case(ek, Fake(), 5000, row)
        sw = ek.debug_program()["sweeps"][0]
    cfg = sw["config"]
    assert cfg["fast"] == 0 and (cfg["V"], cfg["T"], cfg["stages"], cfg["ctas_per_sm"]) == row[3]
    assert lp.general_config(sw, 5000) == row[3]


def test_configuration_table_covers_every_candidate(clean):
    """The test's candidate lists are choose_config's own (as the dry run reports them), and the table covers them all."""
    ek = clean
    cases = lp.live_temps_case(ek, Fake(), 5000, 2)
    configs = ek.debug_program()["configs"]
    assert [tuple(c) for c in configs["wide"]] == lp.WIDE
    assert [tuple(c) for c in configs["small"]] == lp.SMALL
    assert sorted({r[3] for r in lp.CONFIG_ROWS}) == sorted(lp.WIDE)


@pytest.mark.parametrize("n,want", lp.SMALL_ROWS)
def test_small_configuration_plan(clean, n, want):
    ek = clean
    cases = lp.live_temps_case(ek, Fake(), n, 4, 2)
    cfg = ek.debug_program()["sweeps"][0]["config"]
    assert (cfg["V"], cfg["T"], cfg["stages"]) == want[:3] and cfg["fast"] == 0


def test_split_plans(clean, oracle):
    ek = clean
    put = Fake()
    cases = lp.many_outputs_case(ek, put, 1000)
    prog = ek.debug_program()
    assert len(prog["sweeps"]) >= 2
    assert emulate(ek, oracle, put, cases, prog)
    del cases
    gc.collect()
    for count in (lp.MAX_SCALAR + 1, 2 * lp.MAX_SCALAR + 2):
        put = Fake()
        cases = lp.scalar_case(ek, put, 5000, count)
        prog = ek.debug_program()
        lp.check_scalar_plan(prog, 5000, count)
        assert all("fast" in s for s in prog["sweeps"])
        assert emulate(ek, oracle, put, cases, prog)
        del cases
        gc.collect()
    with lp.fast_mode(ek, False):
        cases = lp.pressure_case(ek, Fake(), 5000)
        assert len(ek.debug_program()["sweeps"]) == 2
    del cases
    gc.collect()
    cases = lp.scatter_split_case(ek, Fake(), 4097)
    assert lp.scatter_halves(ek.debug_program()) >= 2
    del cases
    gc.collect()
    cases = lp.split_reduction_case(ek, Fake(), 5000)
    phases = [s["phase"] for s in ek.debug_program()["sweeps"]]
    assert phases.count(0) >= 2 and 1 in phases
