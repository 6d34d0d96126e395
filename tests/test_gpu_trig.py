"""GPU: the Float32 trigonometric operations tan, cot, asin, acos, atan and atan2 on an H100.  Native results against the
C restatements (tests/trig_oracle.c) on special values and 2^24 random arguments per function; the same programs on both
sweep kernels, fused with other operations and reductions, with literal and scalar operands, at ragged sizes and in a sweep
that a 64-bit value forces onto the general kernel; Float16 storage; FloatD gradients; and tests/cpp/trig_check, which
compares every Float32 input with array_math.h's traced bodies on the device."""
import os
import subprocess

import numpy as np
import pytest

import trig_support as ts

HERE = os.path.dirname(os.path.abspath(__file__))
UNARY = ("tan", "cot", "asin", "acos", "atan")
pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def fast_mode(ek, gpu):
    yield
    ek.lib().ek_set_fast_mode(1)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _specials():
    v = np.array([0x00000000, 0x00000001, 0x007fffff, 0x00800000, 0x3f800000, 0x3f000000, 0x3effffff, 0x3f000001,
                  0x3f7fffff, 0x3f800001, 0x7f7fffff, 0x7f800000, 0x7fc00000, 0x7fa00000, 0x38d1b717, 0x38d1b716,
                  0x4f000000, 0x4effffff, 0x46000000, 0x46000001], np.uint32)
    br = (np.arange(1, 200) * np.pi / 4).astype(np.float32).view(np.uint32)
    v = np.concatenate([v, br - 1, br, br + 1])
    return np.concatenate([v, v | np.uint32(0x80000000)]).view(np.float32)


def _random(seed, n):
    rng = np.random.default_rng(seed)
    r = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
    r[: n // 4] = rng.uniform(-1.2, 1.2, n // 4).astype(np.float32)
    r[n // 4: 2 * (n // 4)] = rng.uniform(-50, 50, n // 4).astype(np.float32)
    return r


@pytest.mark.parametrize("name", UNARY)
def test_native_equals_restatement(ek, name):
    x = np.concatenate([_specials(), _random(11, 1 << 24)])
    got = getattr(ek, name)(ek.Float32.copy(x)).numpy()
    ok = ts.same_bits(got, ts.unary(name, x))
    assert ok.all(), (name, x[~ok][:5], got[~ok][:5])


def test_native_atan2_equals_restatement(ek):
    s = np.array([0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, -1.0, 1.0, 0.5, -3.0, 3.4028235e38, np.inf, -np.inf, np.nan], np.float32)
    ys, xs = (a.ravel() for a in np.meshgrid(s, s, indexing="ij"))
    y = np.concatenate([ys, _random(12, 1 << 24)]); x = np.concatenate([xs, _random(13, 1 << 24)])
    got = ek.atan2(ek.Float32.copy(y), ek.Float32.copy(x)).numpy()
    ok = ts.same_bits(got, ts.atan2(y, x))
    assert ok.all(), (y[~ok][:5], x[~ok][:5], got[~ok][:5])


def _program(ek, F, a, b, c, lit_y, lit_x, scalar):
    """every function fused with other operations: literal and scalar operands of atan2 in both positions"""
    t = ek.tan(a * 0.5) + ek.cot(b) * c
    u = ek.asin(ek.select(abs(c) < 1.0, c, c * 0.25)) - ek.acos(ek.min_(ek.max_(a, F(-1.0)), F(1.0)))
    v = ek.atan(t) * ek.atan2(a, b) + ek.atan2(F(lit_y), c) - ek.atan2(b, F(lit_x)) + ek.atan2(scalar, a) * ek.atan2(c, scalar)
    return u + v, ek.hsum(v), ek.hmax(u)


@pytest.mark.parametrize("n", [1, 31, 4097, (1 << 20) + 3])
def test_both_kernels_agree_bit_for_bit(ek, n):
    rng = np.random.default_rng(n)
    data = [rng.uniform(-3, 3, n).astype(np.float32) for _ in range(3)]
    data[0][: max(n // 100, 1)] = np.nan
    results = []
    for fast in (0, 1):
        ek.lib().ek_set_fast_mode(fast)
        F = ek.Float32
        a, b, c = (F.copy(d) for d in data)
        scalar = F.copy(np.array([0.3], np.float32))
        before = int(ek.stats().fast_launches)
        out, s, m = _program(ek, F, a, b, c, -0.75, 2.0, scalar)
        o = out.numpy(); sv = s.numpy(); mv = m.numpy()
        used = int(ek.stats().fast_launches) - before
        if n > 4096:
            assert (used > 0) == (fast == 1), (fast, used)
        results.append((o, sv, mv))
    (o0, s0, m0), (o1, s1, m1) = results
    assert (_bits(o0) == _bits(o1)).all()
    assert _bits(m0) == _bits(m1)
    if n <= 4096:
        assert _bits(s0) == _bits(s1)
    else:                                    # reductions fold partials in a kernel-specific order
        assert np.allclose(s0, s1, rtol=1e-5, atol=1e-3, equal_nan=True)


def test_sweep_with_a_64bit_value_runs_on_the_general_kernel(ek):
    n = (1 << 20) + 3
    x = _random(21, n); y = _random(22, n)
    before = int(ek.stats().fast_launches)
    X, Y = ek.Float32.copy(x), ek.Float32.copy(y)
    wide = ek.Float64(ek.atan2(Y, X)) * 2.0                     # a Float64 value in the same sweep
    r = ek.tan(X) + ek.asin(Y)
    got_w = wide.numpy(); got_r = r.numpy()
    assert int(ek.stats().fast_launches) == before
    want = ts.atan2(y, x)
    assert ts.same_bits((got_w / 2).astype(np.float32), want).all()
    with np.errstate(all="ignore"):
        assert ts.same_bits(got_r, (ts.unary("tan", x) + ts.unary("asin", y)).astype(np.float32)).all()


def test_float16_storage_with_atan2(ek):
    n = (1 << 20) + 5
    rng = np.random.default_rng(5)
    y = rng.uniform(-4, 4, n).astype(np.float16); x = rng.uniform(-4, 4, n).astype(np.float16)
    before = int(ek.stats().fast_launches)
    r = ek.Float16(ek.atan2(ek.Float32(ek.Float16.copy(y)), ek.Float32(ek.Float16.copy(x)))).numpy()
    assert int(ek.stats().fast_launches) > before
    want = ts.atan2(y.astype(np.float32), x.astype(np.float32)).astype(np.float16)
    assert (r.view(np.uint16) == want.view(np.uint16)).all()


def test_floatd_gradients_are_the_appendix_b_weights(ek):
    from enoki_b200 import autodiff as ad
    n = 4099
    rng = np.random.default_rng(9)
    xv = rng.uniform(-0.9, 0.9, n).astype(np.float32); yv = rng.uniform(0.3, 2.0, n).astype(np.float32)
    F = ek.Float32
    for name in UNARY + ("atan2",):
        x = ad.FloatD(F.copy(xv)); y = ad.FloatD(F.copy(yv))
        ad.set_requires_gradient(x); ad.set_requires_gradient(y)
        z = ad.atan2(y, x) if name == "atan2" else getattr(ad, name)(x)
        ad.backward(ad.hsum(z))
        gx = ad.gradient(x).numpy()
        X, Y = F.copy(xv), F.copy(yv)
        if name == "tan":
            s = ek.rcp(ek.cos(X)); want = (s * s).numpy()
        elif name == "cot":
            c = ek.rcp(ek.sin(X)); want = (-(c * c)).numpy()
        elif name == "asin":
            want = ek.rsqrt(1.0 - X * X).numpy()
        elif name == "acos":
            want = (-ek.rsqrt(1.0 - X * X)).numpy()
        elif name == "atan":
            want = ek.rcp(1.0 + X * X).numpy()
        else:
            il2 = ek.rcp(Y * Y + X * X)
            want = (-il2 * Y).numpy()
            gy = ad.gradient(y).numpy()
            assert (_bits(gy) == _bits((il2 * X).numpy())).all()
        assert (_bits(gx) == _bits(want)).all(), name
        assert (_bits(z.numpy()) == _bits((ek.atan2(Y, X) if name == "atan2" else getattr(ek, name)(X)).numpy())).all()


def test_cpp_trig_check(gpu):
    exe = os.path.join(HERE, "cpp", "trig_check")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/trig_check is built only where the reference headers exist")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1800)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "trig_check ok" in r.stdout
