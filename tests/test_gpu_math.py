"""GPU: the Float32 operations pow, frexp, hypot, dawson and erfi on an H100.  Native results against the C
restatements (tests/math_oracle.c) and the reference CPU path's golden vectors (tests/golden/math.npz); the same
programs on both sweep kernels at ragged sizes, with misaligned inputs, with literal and scalar operands in both
positions, in a sweep that a 64-bit value forces onto the general kernel, and with Float16 storage; and
tests/cpp/math_check, which compares the native operations with the traced bodies of array_math.h and special.h on the
device."""
import os
import subprocess

import numpy as np
import pytest

import math_support as ms

HERE = os.path.dirname(os.path.abspath(__file__))
BINARY, UNARY = ms.BINARY, ms.UNARY
pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def fast_mode(ek, gpu):
    yield
    ek.lib().ek_set_fast_mode(1)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _call(ek, name, *args):
    if name in ("frexp_m", "frexp_e"):
        return ek.frexp(*args)[name == "frexp_e"]
    return getattr(ek, {"pow": "pow_"}.get(name, name))(*args)


def _check(got, want, what):
    """raw bits where the restatement's result is not NaN (the device's NaNs are canonical, x86 propagates payloads),
    NaN where it is"""
    ok = ms.same_bits(got, want)
    assert ok.all(), (what, int((~ok).sum()), _bits(got)[~ok][:5], _bits(want)[~ok][:5])


def _pairs(seed, n):
    rng = np.random.default_rng(seed)
    x, y = rng.integers(0, 1 << 32, (2, n), dtype=np.uint64).astype(np.uint32).view(np.float32)
    q = n // 4
    x[:q] = rng.uniform(0, 10, q); y[:q] = rng.uniform(-8, 8, q)
    x[q:2 * q] = rng.uniform(-12, 12, q); y[q:2 * q] = rng.uniform(-12, 12, q)
    return x, y


@pytest.mark.parametrize("name", BINARY + UNARY)
def test_native_equals_restatement_and_golden(ek, name):
    d = np.load(os.path.join(HERE, "golden", "math.npz"))
    if name in BINARY:
        gx, gy = d["bx"], d["by"]
        got = _call(ek, name, ek.Float32.copy(gx), ek.Float32.copy(gy)).numpy()
        rx, ry = _pairs(51 + BINARY.index(name), 1 << 22)
        before = int(ek.stats().fast_launches)
        rgot = _call(ek, name, ek.Float32.copy(rx), ek.Float32.copy(ry)).numpy()
        assert int(ek.stats().fast_launches) > before
        _check(rgot, ms.binary(name, rx, ry), name)
        want = ms.binary(name, gx, gy)
    else:
        gx = d["x"]
        got = _call(ek, name, ek.Float32.copy(gx)).numpy()
        want = ms.unary(name, gx)
    _check(got, want, name)
    _check(got, d[name], name + " (reference CPU path)")


def _program(ek, a, b, s):
    """every function, fused with other operations, literal and scalar operands in both positions"""
    m, e = ek.frexp(a * 3.0)
    t = ek.pow_(ek.abs_(a), 2.2) + ek.pow_(1.5, b * 0.5) + m * e
    u = ek.hypot(a, 2.0) * ek.hypot(s, b * 1.0) - ek.hypot(3.0, b * 0.5)
    v = ek.dawson(t * 0.1) + ek.erfi(u * 0.25) + ek.pow_(s, a * 1.0) + ek.hypot(b * 2.0, a)
    return t + u, v, ek.hsum(v), ek.hmax(t)


def _program_ref(a, b, s):
    f = np.float32
    B, U = ms.binary, ms.unary
    with np.errstate(all="ignore"):
        a3 = (a * f(3)).astype(f)
        m, e = U("frexp_m", a3), U("frexp_e", a3)
        t = ((B("pow", np.abs(a), f(2.2)) + B("pow", f(1.5), (b * f(0.5)).astype(f))).astype(f)
             + (m * e).astype(f)).astype(f)
        u = ((B("hypot", a, f(2)) * B("hypot", s, (b * f(1)).astype(f))).astype(f)
             - B("hypot", f(3), (b * f(0.5)).astype(f))).astype(f)
        v = (((U("dawson", (t * f(0.1)).astype(f)) + U("erfi", (u * f(0.25)).astype(f))).astype(f)
              + B("pow", s, (a * f(1)).astype(f))).astype(f) + B("hypot", (b * f(2)).astype(f), a)).astype(f)
        return (t + u).astype(f), v


@pytest.mark.parametrize("n", [1, 4097, (1 << 20) + 7])
def test_both_kernels_agree_bit_for_bit(ek, n):
    rng = np.random.default_rng(n)
    data = [rng.uniform(-4, 4, n).astype(np.float32) for _ in range(2)]
    data[0][: max(n // 100, 1)] = np.nan
    results = []
    for fast in (0, 1):
        ek.lib().ek_set_fast_mode(fast)
        a, b = (ek.Float32.copy(d) for d in data)
        s = ek.Float32.copy(np.array([0.75], np.float32))
        before = int(ek.stats().fast_launches)
        o, v, sv, mv = (r.numpy() for r in _program(ek, a, b, s))
        used = int(ek.stats().fast_launches) - before
        if n > 4096:
            assert (used > 0) == (fast == 1), (fast, used)
        results.append((o, v, sv, mv))
    (o0, v0, s0, m0), (o1, v1, s1, m1) = results
    assert (_bits(o0) == _bits(o1)).all() and (_bits(v0) == _bits(v1)).all()
    assert _bits(m0) == _bits(m1)
    if n <= 4096:
        assert _bits(s0) == _bits(s1)
    else:                                    # reductions fold partials in a kernel-specific order
        assert np.allclose(s0, s1, rtol=1e-4, atol=1e-2, equal_nan=True)
    wo, wv = _program_ref(data[0], data[1], np.float32(0.75))
    _check(o1, wo, "t + u")
    _check(v1, wv, "v")


def test_misaligned_inputs(ek):
    """inputs mapped one element past a 16-byte aligned base (staged without TMA), on the fast kernel"""
    from test_gpu_horizontal import Staging
    n = (1 << 20) + 3
    x, y = _pairs(71, n)
    put = Staging(ek, "misaligned")
    try:
        X, Y = put(ek.Float32, x, np.float32([0])), put(ek.Float32, y, np.float32([0]))
        before = int(ek.stats().fast_launches)
        for name in BINARY:
            _check(_call(ek, name, X, Y).numpy(), ms.binary(name, x, y), name)
        for name in UNARY:
            _check(_call(ek, name, Y).numpy(), ms.unary(name, y), name)
        assert int(ek.stats().fast_launches) > before
    finally:
        put.free()


def test_sweep_with_a_64bit_value_runs_on_the_general_kernel(ek):
    n = (1 << 20) + 7
    x, y = _pairs(61, n)
    before = int(ek.stats().fast_launches)
    X, Y = ek.Float32.copy(x), ek.Float32.copy(y)
    wide = ek.Float64(ek.dawson(X)) * 2.0                    # a Float64 value in the same sweep
    m, e = ek.frexp(X)
    r = [ek.pow_(X, Y), ek.hypot(X, Y), ek.pow_(Y, X * 1.0), ek.hypot(Y, X * 1.0), m, e, ek.erfi(Y)]
    got = [v.numpy() for v in r]
    got_w = wide.numpy()
    assert int(ek.stats().fast_launches) == before
    assert ms.same_bits((got_w / 2).astype(np.float32), ms.unary("dawson", x)).all()
    want = [ms.binary("pow", x, y), ms.binary("hypot", x, y), ms.binary("pow", y, x), ms.binary("hypot", y, x),
            ms.unary("frexp_m", x), ms.unary("frexp_e", x), ms.unary("erfi", y)]
    for k, (g, w) in enumerate(zip(got, want)):
        _check(g, w, k)


def test_float16_storage(ek):
    n = (1 << 20) + 5
    rng = np.random.default_rng(6)
    x, y = (rng.uniform(-4, 4, n).astype(np.float16) for _ in range(2))
    before = int(ek.stats().fast_launches)
    X, Y = ek.Float32(ek.Float16.copy(x)), ek.Float32(ek.Float16.copy(y))
    r = ek.Float16(ek.hypot(X, Y) + ek.pow_(ek.abs_(X), 1.5) + ek.dawson(Y)).numpy()
    assert int(ek.stats().fast_launches) > before
    xf, yf = x.astype(np.float32), y.astype(np.float32)
    with np.errstate(all="ignore"):
        want = ((ms.binary("hypot", xf, yf) + ms.binary("pow", np.abs(xf), np.float32(1.5))).astype(np.float32)
                + ms.unary("dawson", yf)).astype(np.float32).astype(np.float16)
    assert (r.view(np.uint16) == want.view(np.uint16)).all()


def test_cpp_math_check(gpu):
    exe = os.path.join(HERE, "cpp", "math_check")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/math_check is built only where the reference headers exist")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1800)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "math_check ok" in r.stdout
