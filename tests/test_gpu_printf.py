"""GPU: cuda_printf end to end, the printed text checked exactly.

Every expected line comes from the C library's own snprintf (through ctypes) applied to values computed on the host
with operations that numpy reproduces bit for bit, each value converted to the C type its conversion names.  The
lines are read from file descriptor 1 (capfd): the evaluation writes them before it returns."""
import ctypes
import gc
import os
import re
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_libc = ctypes.CDLL(None)
_libc.snprintf.restype = ctypes.c_int
_BUF = ctypes.create_string_buffer(1 << 14)
_CONV = re.compile(r"%[-+ #0]*\d*(?:\.\d*)?(hh|h|ll|l)?([diuoxXcfFeEgGaA%])")
_INT_CTYPE = {"d": (ctypes.c_int, ctypes.c_long, ctypes.c_longlong), "u": (ctypes.c_uint, ctypes.c_ulong, ctypes.c_ulonglong)}


def ctypes_of(fmt):
    """The C type each conversion of `fmt` takes (what C's printf reads for it)."""
    out = []
    for m in _CONV.finditer(fmt):
        length, conv = m.group(1) or "", m.group(2)
        if conv == "%":
            continue
        if conv in "fFeEgGaA":
            out.append(ctypes.c_double)
        else:
            k = 2 if length == "ll" else 1 if length == "l" else 0
            out.append(_INT_CTYPE["d" if conv in "dic" else "u"][k])
    return out


def c_line(fmt, cts, values):
    args = [ct(float(v) if ct is ctypes.c_double else int(v)) for ct, v in zip(cts, values)]
    n = _libc.snprintf(_BUF, len(_BUF), fmt.encode(), *args)
    assert 0 <= n < len(_BUF)
    return _BUF.raw[:n].decode()


def expect(fmt, *arrays, n=None):
    """The text of one print: a line per element, size-1 arrays broadcast."""
    arrays = [np.atleast_1d(np.asarray(a)) for a in arrays]
    n = n if n is not None else max([len(a) for a in arrays] or [1])
    cts = ctypes_of(fmt)
    assert len(cts) == len(arrays)
    return "".join(c_line(fmt, cts, [a[0 if len(a) == 1 else i] for a in arrays]) for i in range(n))


@pytest.fixture()
def ek():
    import enoki_b200 as ek
    if ek.device_count() == 0:
        pytest.fail("GPU test selected but no CUDA device is visible (there is no CPU fallback)")
    gc.collect()
    assert ek.debug_plan() == ""
    yield ek
    gc.collect()
    assert ek.debug_plan() == "", "a print (or its arguments) is still recorded after the evaluation"


def evaluate(ek, capfd):
    capfd.readouterr()
    ek.cuda_eval()
    return capfd.readouterr().out


INT_VALUES = {
    "Int8": [0, 1, -1, 127, -128, 42, -42],
    "UInt8": [0, 1, 255, 128, 127, 42],
    "Int16": [0, 1, -1, 32767, -32768, 1234, -1234],
    "UInt16": [0, 1, 65535, 32768, 4321],
    "Int32": [0, 1, -1, 2**31 - 1, -2**31, 123456789, -987654321],
    "UInt32": [0, 1, 2**32 - 1, 2**31, 2**31 - 1, 3000000000],
    "Int64": [0, 1, -1, 2**63 - 1, -2**63, 2**32, -2**40 - 3],
    "UInt64": [0, 1, 2**64 - 1, 2**63, 2**32 + 5, 12345678901234567890],
    "Mask": [True, False, True, True],
}
INT_FORMATS = ["%d %i %u\n", "%x %X %o\n", "%hhd %hhu %hx\n", "%hd %hi %hX\n", "%ld %lu %lx\n", "%lld %llu %llo\n",
               "%+d|%-8i|%08x\n", "%#o %#X % d\n", "%.3d %5.2u %-#10x|\n", "%+.0d|%20llu|%-20lld|\n", "%%%d%%%i%%%u%%\n"]


@pytest.mark.parametrize("tname", list(INT_VALUES))
def test_integer_conversions(ek, capfd, tname):
    cls = getattr(ek, tname)
    xs = np.array(INT_VALUES[tname], dtype=ek._NP[cls.Type])
    x = cls.copy(xs)
    y = ~x if tname == "Mask" else x ^ cls(1)          # computed: stored by its sweep for the print
    ys = ~xs if tname == "Mask" else xs ^ xs.dtype.type(1)
    want = ""
    for fmt in INT_FORMATS:
        ek.cuda_printf(fmt, x, x, x)
        want += expect(fmt, xs, xs, xs)
        ek.cuda_printf(fmt, y, x, y)
        want += expect(fmt, ys, xs, ys)
    del y
    assert evaluate(ek, capfd) == want


F32_VALUES = [0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 1.0, -1.5, 1 / 3, 1e-45, -1.4e-40, 3.4028235e38, 1.1754944e-38,
              123456.789, 2.5, -2.5, 0.1]
F64_VALUES = F32_VALUES + [5e-324, -1e-310, 1.7976931348623157e308, 2.2250738585072014e-308, 1 / 3, -0.1]
FLOAT_FORMATS = ["%f %e %g\n", "%.3f|%-14.5e|%+G\n", "%#a %A %12.4E\n", "%F % .0f %010.2lf\n",
                 "%.17g %#.0e %-+8.1f|\n", "%.9g %lg %.1a\n", "%5.0f %#g %-.3G|\n"]


@pytest.mark.parametrize("tname", ["Float32", "Float64"])
def test_float_conversions(ek, capfd, tname):
    cls = getattr(ek, tname)
    xs = np.array(F32_VALUES if tname == "Float32" else F64_VALUES, dtype=ek._NP[cls.Type])
    x = cls.copy(xs)
    zs = np.where(np.isnan(xs), xs.dtype.type(0), xs)  # (a negated NaN's sign is not part of the contract of NEG)
    y = -cls.copy(zs)
    ys = -zs
    want = ""
    for fmt in FLOAT_FORMATS:
        ek.cuda_printf(fmt, x, y, x)
        want += expect(fmt, xs, ys, xs)
    del y
    assert evaluate(ek, capfd) == want


def test_char_conversion(ek, capfd):
    xs = np.arange(65, 91, dtype=np.uint32)
    x = ek.UInt32.copy(xs)
    c = ek.Int8(x - 32)
    ek.cuda_printf("%c%-3c|%2c\n", x, c, ek.Mask(True))
    del c
    assert evaluate(ek, capfd) == expect("%c%-3c|%2c\n", xs, (xs - 32).astype(np.int8), [1])


def test_pointer_arguments(ek, capfd):
    L = ek.lib()
    vals = np.array([0, 0xdeadbeef, 2**64 - 1, 0x7f0000001000], np.uint64)
    u = ek.UInt64.copy(vals).eval()
    arr = L.ek_var_register(ek.EK_POINTER, 4, L.ek_var_ptr(u.index), 0)       # a pointer array aliasing u
    reg = L.ek_var_register_ptr(ctypes.c_void_p(0x12345678))                   # a registered pointer (size 1)
    try:
        fmt = "%lx %llu %#lX\n"
        assert L.ek_trace_printf(fmt.encode(), 3, (ctypes.c_uint32 * 3)(arr, arr, reg)) == 0, L.ek_last_error()
    finally:
        L.ek_dec_ref_ext(arr)
        L.ek_dec_ref_ext(reg)
    assert evaluate(ek, capfd) == expect(fmt, vals, vals, [0x12345678])


def test_size1_literal_and_zero_argument_prints(ek, capfd):
    ek.cuda_printf("no arguments\n")
    ek.cuda_printf("%d %f %u\n", ek.Int32(-7), ek.Float64(2.5), ek.UInt8(200))
    s = ek.Float32(1.5) * ek.Float32(3.0)
    ek.cuda_printf("%f\n", s)
    w = ek.Float32.full(1.25, 3)
    ek.cuda_printf("%g|\n", w)
    r = ek.hsum(ek.UInt32.arange(100))
    ek.cuda_printf("%u %u\n", r, ek.UInt32.arange(4))
    del s, w, r
    want = ("no arguments\n" + expect("%d %f %u\n", [-7], [2.5], [200]) + expect("%f\n", np.float32(4.5)) +
            expect("%g|\n", np.float32(1.25), n=3) + expect("%u %u\n", [4950], np.arange(4)))
    assert evaluate(ek, capfd) == want


@pytest.mark.parametrize("n", [1, 31, 4097, 2049])
def test_ragged_sizes(ek, capfd, n):
    """1 and 31: one small CTA; 4097: one fast-kernel tile (256 x 16) + 1; 2049: one general-kernel tile (256 x 8) + 1,
    the print of a Float64 value sending the sweep there."""
    xs = (np.arange(n, dtype=np.uint32) * np.uint32(2654435761)).astype(np.uint32)
    x = ek.UInt32.copy(xs)
    y = x * 3 + 1
    ys = xs * np.uint32(3) + np.uint32(1)
    if n == 2049:
        f = ek.Float64(x) * 0.5
        fs = xs.astype(np.float64) * 0.5
        ek.cuda_printf("%u %u %.1f\n", x, y, f)
        want = expect("%u %u %.1f\n", xs, ys, fs)
        del f
    else:
        ek.cuda_printf("%u %08x\n", x, y)
        want = expect("%u %08x\n", xs, ys)
    del y
    out = evaluate(ek, capfd)
    assert out.count("\n") == n and out == want


def test_order_of_prints(ek, capfd):
    """Two prints of one size and one of another size between them: recording order, whatever the launch order."""
    a = ek.UInt32.arange(10) + 100
    c = ek.UInt32.arange(5) * 7
    b = ek.UInt32.arange(10) + 300
    ek.cuda_printf("A %u\n", a)
    ek.cuda_printf("C %u\n", c)
    ek.cuda_printf("B %u\n", b)
    want = (expect("A %u\n", np.arange(10) + 100) + expect("C %u\n", np.arange(5) * 7) +
            expect("B %u\n", np.arange(10) + 300))
    assert evaluate(ek, capfd) == want
    assert np.array_equal(b.numpy(), np.arange(10) + 300)


def test_value_at_recording(ek, capfd):
    """A scatter recorded after the print, in the same evaluation, writes into the printed array."""
    xs = np.arange(10, dtype=np.uint32) * 3
    x = ek.UInt32.copy(xs)
    ek.cuda_printf("%u\n", x)
    ek.scatter(x, ek.UInt32(99), ek.UInt32.arange(10))
    assert evaluate(ek, capfd) == expect("%u\n", xs)
    assert np.array_equal(x.numpy(), np.full(10, 99, np.uint32))
    # a dirty argument is evaluated first: the print shows what the scatter wrote
    ek.scatter(x, ek.UInt32(5), ek.UInt32.arange(4))
    ek.cuda_printf("%u\n", x)
    assert evaluate(ek, capfd) == expect("%u\n", np.array([5] * 4 + [99] * 6))


def program(ek, x):
    t = ek.fmadd(x, ek.Float32(1.5), ek.Float32(0.25))
    z = ek.sin(t) * ek.exp(-(x * x)) + t
    return t, z


def test_intermediate_and_other_outputs(ek, capfd):
    """The print of an intermediate that nothing else stores; the program's own output is bit-identical with and
    without the print."""
    xs = np.random.default_rng(3).standard_normal(5000).astype(np.float32)
    x = ek.Float32.copy(xs)
    _t, z = program(ek, x)
    del _t
    plain = z.numpy()
    assert evaluate(ek, capfd) == ""
    k = ek.UInt32.arange(5000)
    m = k * 5 + 2                                     # bit-exact integer intermediate, stored nowhere else
    t, z = program(ek, x)
    ek.cuda_printf("%u %a\n", m, t)
    del m
    out = evaluate(ek, capfd)
    ts = t.numpy()
    assert out == expect("%u %a\n", np.arange(5000, dtype=np.uint32) * 5 + 2, ts)
    assert np.array_equal(z.numpy().view(np.uint32), plain.view(np.uint32))


@pytest.mark.parametrize("tname,fast", [("UInt32", 1), ("Float32", 1), ("Mask", 1), ("Int16", 0), ("Float64", 0), ("Int64", 0)])
def test_kernel_choice(ek, capfd, tname, fast):
    """A 32-bit program that prints stays on the fast kernel (ST_32 / ST_8); a 16- or 64-bit print goes to the general
    kernel, as a store of such a value does."""
    assert ek.lib().ek_fast_mode() == 1
    cls = ek.UInt32 if tname == "Mask" else getattr(ek, tname)
    xs = (np.arange(5000) % 100).astype(ek._NP[cls.Type])
    x = cls.copy(xs)
    y = x < 50 if tname == "Mask" else x + cls(3)
    ys = xs < 50 if tname == "Mask" else xs + xs.dtype.type(3)
    fmt = "%f\n" if tname.startswith("Float") else "%d\n"
    ek.cuda_printf(fmt, y)
    del y
    ek.lib().ek_stats_reset()
    assert evaluate(ek, capfd) == expect(fmt, ys)
    st = ek.stats()
    assert st.sweep_launches == 1 and st.fast_launches == fast


def test_one_million_lines(ek, capfd):
    n = 1 << 20
    k = ek.UInt32.arange(n)
    y = ek.Float32(k) * 0.5
    ek.cuda_printf("%u %.1f\n", k, y)
    del k, y
    out = evaluate(ek, capfd)
    ks = np.arange(n, dtype=np.uint32)
    assert out == expect("%u %.1f\n", ks, ks.astype(np.float32) * np.float32(0.5))


def test_rejected_format_on_gpu(ek, capfd):
    x = ek.Float32.copy(np.arange(4, dtype=np.float32))
    with pytest.raises(ek.EnokiError, match="'%d'.*f32"):
        ek.cuda_printf("%d\n", x)
    assert evaluate(ek, capfd) == ""


def test_cpp_printf_check(gpu):
    """The reference's cuda_printf template over CUDAArray<float> / CUDAArray<uint32_t> (tests/cpp/printf_check.cpp)."""
    binp = os.path.join(ROOT, "tests", "cpp", "printf_check")
    if not os.path.exists(binp):
        pytest.skip("tests/cpp/printf_check not built (needs the reference headers at build time)")
    r = subprocess.run([binp], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "all checks passed" in r.stderr
    i = np.arange(11, dtype=np.uint32)
    x = i.astype(np.float32) * np.float32(0.125)
    y = x * x + np.float32(1)
    want = (expect("i=%u x=%f y=%.4e\n", i, x, y) + expect("scalar %u\n", [7]) + "no arguments\n" +
            expect("%u %g\n", i[:3] * np.uint32(3), [np.float32(0.5)]))
    assert r.stdout.splitlines() == want.splitlines()
