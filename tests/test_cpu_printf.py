"""CPU: cuda_printf's recording side, checked without a GPU.

A print is checked when it is recorded (a rejected format or argument list records nothing), the dry run lists each
print with its format, arguments and size, and a computed argument is stored by the sweep that computes it: the
program the planner builds for a print of an intermediate value runs on the numpy interpreter of the sweep ISA
(tests/ek_emulator.py) and stores exactly the argument's values, and a print of a value the sweep stores anyway
changes nothing in the sweep."""
import ctypes
import gc

import numpy as np
import pytest

from ek_emulator import Emulator


class Fake:
    """put(cls, array): a fake device mapping whose data the emulator reads."""
    def __init__(self):
        self.table, self.k = {}, 0

    def __call__(self, cls, arr):
        self.k += 1
        r = cls.map(0x700000000000 + 0x10000000 * self.k, len(arr))
        self.table[r.index] = np.ascontiguousarray(arr)
        return r


@pytest.fixture()
def clean(ek):
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()
    assert ek.debug_plan() == "", "unevaluated variables of an earlier test are still alive"
    yield ek
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()
    assert ek.debug_plan() == ""


def raw_printf(ek, fmt, *handles):
    """ek_trace_printf on raw handles (0 = uninitialised); returns (rc, message)."""
    L = ek.lib()
    arr = (ctypes.c_uint32 * max(len(handles), 1))(*handles)
    rc = L.ek_trace_printf(fmt.encode(), len(handles), arr)
    return rc, L.ek_last_error().decode()


REJECTED = [
    # (format, argument types, words the message must contain)
    ("%s", ["Float32"], ["'%s'", "f32"]),
    ("%n", ["UInt32"], ["'%n'", "u32"]),
    ("%p", ["UInt64"], ["'%p'", "u64"]),
    ("%d", ["Float32"], ["'%d'", "f32"]),
    ("%x", ["Float64"], ["'%x'", "f64"]),
    ("%f", ["UInt32"], ["'%f'", "u32"]),
    ("%e", ["Int64"], ["'%e'", "i64"]),
    ("%g", ["Mask"], ["'%g'", "bool"]),
    ("%d %d", ["Int32"], ["'%d'", "no argument"]),
    ("%d", ["Int32", "Int32"], ["1 conversion", "2 argument"]),
    ("no conversion", ["Float32"], ["0 conversion", "1 argument"]),
    ("%u", [], ["'%u'", "no argument"]),
    ("value %", ["Int32"], ["lone '%'"]),
    ("%", [], ["lone '%'"]),
    ("%5", ["Int32"], ["ends inside", "'%5'"]),
    ("%*d", ["Int32"], ["'*'", "i32"]),
    ("%.*f", ["Float32"], ["'*'", "f32"]),
    ("%Lf", ["Float64"], ["'%L'", "f64"]),
    ("%zu", ["UInt64"], ["'%z'", "u64"]),
    ("%jd", ["Int64"], ["'%j'", "i64"]),
    ("%hf", ["Float32"], ["'%hf'", "'h'", "f32"]),
    ("%llg", ["Float64"], ["'%llg'", "'ll'", "f64"]),
    ("%lc", ["Int32"], ["'%lc'", "'l'", "i32"]),
    ("%C", ["Int32"], ["'%C'", "i32"]),
    ("%5000d", ["Int32"], ["width", "4096"]),
    ("%.5000f", ["Float64"], ["precision", "4096"]),
    ("%d %s", ["Int8", "UInt16"], ["'%s'", "u16"]),
]


@pytest.mark.parametrize("fmt,types,words", REJECTED, ids=[r[0] + "|" + ",".join(r[1]) for r in REJECTED])
def test_rejected_format_records_nothing(clean, fmt, types, words):
    ek = clean
    put = Fake()
    args = [put(getattr(ek, t), np.zeros(5, ek._NP[getattr(ek, t).Type])) for t in types]
    before = ek.debug_plan()
    with pytest.raises(ek.EnokiError) as e:
        ek.cuda_printf(fmt, *args)
    for w in words:
        assert w in str(e.value), (w, str(e.value))
    assert ek.debug_plan() == before == ""


def test_rejected_arguments_record_nothing(clean):
    ek = clean
    put = Fake()
    a, b, c, d = (put(ek.Float32, np.zeros(4, np.float32)) for _ in range(4))
    rc, msg = raw_printf(ek, "%f %f %f %f", a.index, b.index, c.index, d.index)
    assert rc == -1 and msg == "cuda_trace_print(): at most 3 variables can be printed at once!"
    assert ek.debug_plan() == ""
    rc, msg = raw_printf(ek, "%f", 0)
    assert rc == -1 and "uninitialized variable" in msg
    rc, msg = raw_printf(ek, "%f", 123456)
    assert rc == -1 and "unknown variable" in msg
    e = put(ek.Float32, np.zeros(7, np.float32))
    with pytest.raises(ek.EnokiError, match=r"incompatible size \(4 and 7\)"):
        ek.cuda_printf("%f %f", a, e)
    L = ek.lib()
    h = L.ek_var_register(ek.EK_FLOAT16, 4, ctypes.c_void_p(0x7f0000000000), 0)
    try:
        rc, msg = raw_printf(ek, "%f", h)
        assert rc == -1 and "f16" in msg
    finally:
        L.ek_dec_ref_ext(h)
    assert ek.debug_plan() == ""


def test_prints_listing(clean):
    ek = clean
    put = Fake()
    x = put(ek.Float32, np.arange(10, dtype=np.float32))
    k = put(ek.UInt32, np.arange(10, dtype=np.uint32))
    y = x * 2.0
    ek.cuda_printf("x=%f y=%.3e k=%u\n", x, y, k)
    ek.cuda_printf("scalar %d\n", ek.Int32(-3))
    ek.cuda_printf("no arguments\n")
    s = ek.Float32(1.5) + ek.Float32(2.0)           # computed size-1 value broadcast against a wide one
    ek.cuda_printf("%g %f\n", s, y)
    prog = ek.debug_program()
    prints = prog["prints"]
    assert [p["fmt"] for p in prints] == ["x=%f y=%.3e k=%u\n", "scalar %d\n", "no arguments\n", "%g %f\n"]
    assert [p["size"] for p in prints] == [10, 1, 1, 10]
    assert prints[0]["args"] == [x.index, y.index, k.index]
    assert prints[2]["args"] == []
    assert prints[3]["args"] == [s.index, y.index]
    outputs = {o[0] for sw in prog["sweeps"] for o in sw["outputs"]}
    assert {y.index, s.index} <= outputs
    assert x.index not in outputs and k.index not in outputs
    plan = ek.debug_plan()
    assert plan.count("print n=") == 4 and 'fmt="no arguments\\n"' in plan
    # a print of evaluated and literal values only plans no sweep
    del y, s
    gc.collect()
    ek.lib().ek_debug_discard_side_effects()
    ek.cuda_printf("%f %u %d\n", x, k, ek.Int32(7))
    prog = ek.debug_program()
    assert prog["sweeps"] == [] and len(prog["prints"]) == 1


def test_print_of_intermediate_is_stored(clean, oracle):
    """t = x * 3 + k is consumed by z and printed, but referenced by nothing else: the sweep stores it for the print."""
    ek = clean
    put = Fake()
    rng = np.random.default_rng(5)
    xs = rng.standard_normal(5000).astype(np.float32)
    ks = rng.integers(0, 1000, 5000).astype(np.float32)
    x, k = put(ek.Float32, xs), put(ek.Float32, ks)
    t = x * 3.0 + k
    z = ek.sqrt(abs(t)) * t
    ti = t.index
    ek.cuda_printf("%a\n", t)
    del t
    gc.collect()
    prog = ek.debug_program()
    assert prog["prints"][0]["args"] == [ti]
    sw = prog["sweeps"]
    assert len(sw) == 1 and ti in [o[0] for o in sw[0]["outputs"]]
    assert "fast" in sw[0]
    emu = Emulator(oracle, put.table)
    emu.run(prog)
    want = xs * np.float32(3.0) + ks
    got = np.ascontiguousarray(emu.vars[ti]).reshape(-1).view(np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    del z


@pytest.mark.parametrize("tname", ["Float32", "UInt32", "Int64", "UInt8"])
def test_print_of_stored_value_adds_nothing(clean, tname):
    ek = clean
    put = Fake()
    cls = getattr(ek, tname)
    x = put(cls, np.arange(5000).astype(ek._NP[cls.Type]))
    y = x * cls(3) + cls(1)
    before = ek.debug_program()["sweeps"]
    ek.cuda_printf("%u\n" if tname != "Float32" else "%f\n", y)
    after = ek.debug_program()
    assert after["sweeps"] == before
    assert after["prints"][0]["args"] == [y.index]
