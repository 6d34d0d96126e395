"""GPU: the Float32 operations sinh, cosh, tanh, asinh, acosh, atanh and cbrt on an H100.  Native results against the C
restatements (tests/hyp_oracle.c) on the golden arguments and 2^24 random arguments per function; the same programs on
both sweep kernels, fused with other operations and reductions, at ragged sizes, in a sweep that a 64-bit value forces
onto the general kernel, and with Float16 storage; FloatD gradients; and tests/cpp/hyp_check, which compares every
Float32 input with array_math.h's traced bodies on the device."""
import os
import subprocess

import numpy as np
import pytest

import hyp_support as hs

HERE = os.path.dirname(os.path.abspath(__file__))
UNARY = hs.UNARY
pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def fast_mode(ek, gpu):
    yield
    ek.lib().ek_set_fast_mode(1)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _random(seed, n):
    rng = np.random.default_rng(seed)
    r = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
    r[: n // 4] = rng.uniform(-2, 2, n // 4).astype(np.float32)
    r[n // 4: 2 * (n // 4)] = rng.uniform(-100, 100, n // 4).astype(np.float32)
    return r


def _check(name, x, got):
    """raw bits where the restatement's result is not NaN (the device's NaNs are canonical, x86 propagates payloads);
    NaN where it is NaN, and acosh's all-ones NaN of x < 1 exactly (a NaN argument gives a NaN of its own)"""
    want = hs.unary(name, x)
    ok = hs.same_bits(got, want) & ((_bits(got) == _bits(want)) | np.isnan(want))
    if name == "acosh":
        below = ~np.isnan(x) & (x < 1)
        ok &= (_bits(got) == 0xffffffff) == below
    assert ok.all(), (name, int((~ok).sum()), x[~ok][:5], _bits(got)[~ok][:5], _bits(want)[~ok][:5])


@pytest.mark.parametrize("name", UNARY)
def test_native_equals_restatement(ek, name):
    x = np.concatenate([np.load(os.path.join(HERE, "golden", "hyp.npz"))["x"], _random(11 + UNARY.index(name), 1 << 24)])
    before = int(ek.stats().fast_launches)
    got = getattr(ek, name)(ek.Float32.copy(x)).numpy()
    assert int(ek.stats().fast_launches) > before
    _check(name, x, got)


def test_sincosh_is_sinh_and_cosh(ek):
    x = _random(12, 1 << 20)
    s, c = ek.sincosh(ek.Float32.copy(x))
    _check("sinh", x, s.numpy())
    _check("cosh", x, c.numpy())


def _program(ek, a, b, c, scalar):
    """every function fused with other operations and a scalar operand"""
    t = ek.sinh(a * 0.5) + ek.cosh(b) * c - ek.tanh(a + b)
    u = ek.asinh(c * 7.0) - ek.acosh(abs(b) + 1.0) + ek.atanh(ek.min_(ek.max_(a, ek.Float32(-0.99)), ek.Float32(0.99)))
    v = ek.cbrt(t * scalar) + ek.cbrt(u) * ek.tanh(scalar)
    return t + v, ek.hsum(v), ek.hmax(u)


def _clamp(a):
    """min_(max_(a, -0.99), 0.99) with the evaluator's operand rule: a NaN gives the second operand"""
    m = np.where(a > np.float32(-0.99), a, np.float32(-0.99))
    return np.where(m < np.float32(0.99), m, np.float32(0.99)).astype(np.float32)


@pytest.mark.parametrize("n", [1, 4097, (1 << 20) + 7])
def test_both_kernels_agree_bit_for_bit(ek, n):
    rng = np.random.default_rng(n)
    data = [rng.uniform(-3, 3, n).astype(np.float32) for _ in range(3)]
    data[0][: max(n // 100, 1)] = np.nan
    results = []
    for fast in (0, 1):
        ek.lib().ek_set_fast_mode(fast)
        a, b, c = (ek.Float32.copy(d) for d in data)
        scalar = ek.Float32.copy(np.array([0.3], np.float32))
        before = int(ek.stats().fast_launches)
        out, s, m = _program(ek, a, b, c, scalar)
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
    # and the element-wise result against the restatements
    a, b, c = data
    with np.errstate(all="ignore"):
        f = np.float32
        t = ((hs.unary("sinh", a * f(0.5)) + hs.unary("cosh", b) * c).astype(f) - hs.unary("tanh", (a + b).astype(f))).astype(f)
        u = ((hs.unary("asinh", (c * f(7)).astype(f)) - hs.unary("acosh", (np.abs(b) + f(1)).astype(f))).astype(f)
             + hs.unary("atanh", _clamp(a))).astype(f)
        v = (hs.unary("cbrt", (t * f(0.3)).astype(f)) + hs.unary("cbrt", u) * hs.unary("tanh", np.array([0.3], f))).astype(f)
        want = (t + v).astype(f)
    assert hs.same_bits(o1, want).all()


def test_sweep_with_a_64bit_value_runs_on_the_general_kernel(ek):
    n = (1 << 20) + 7
    x = _random(21, n)
    before = int(ek.stats().fast_launches)
    X = ek.Float32.copy(x)
    wide = ek.Float64(ek.cbrt(X)) * 2.0                      # a Float64 value in the same sweep
    r = ek.sinh(X) + ek.acosh(X)
    got_w = wide.numpy(); got_r = r.numpy()
    assert int(ek.stats().fast_launches) == before
    assert hs.same_bits((got_w / 2).astype(np.float32), hs.unary("cbrt", x)).all()
    with np.errstate(all="ignore"):
        assert hs.same_bits(got_r, (hs.unary("sinh", x) + hs.unary("acosh", x)).astype(np.float32)).all()


def test_float16_storage(ek):
    n = (1 << 20) + 5
    x = np.random.default_rng(5).uniform(-4, 4, n).astype(np.float16)
    before = int(ek.stats().fast_launches)
    X = ek.Float32(ek.Float16.copy(x))
    r = ek.Float16(ek.tanh(X) + ek.cbrt(X)).numpy()
    assert int(ek.stats().fast_launches) > before
    xf = x.astype(np.float32)
    want = (hs.unary("tanh", xf) + hs.unary("cbrt", xf)).astype(np.float32).astype(np.float16)
    assert (r.view(np.uint16) == want.view(np.uint16)).all()


def test_floatd_gradients_are_the_autodiff_weights(ek):
    from enoki_b200 import autodiff as ad
    n = 4099
    rng = np.random.default_rng(9)
    F = ek.Float32
    for name in UNARY:
        lo, hi = {"acosh": (1.1, 5.0), "atanh": (-0.9, 0.9)}.get(name, (-3.0, 3.0))
        xv = rng.uniform(lo, hi, n).astype(np.float32)
        x = ad.FloatD(F.copy(xv))
        ad.set_requires_gradient(x)
        z = getattr(ad, name)(x)
        ad.backward(ad.hsum(z))
        gx = ad.gradient(x).numpy()
        X = F.copy(xv)
        if name == "sinh":
            want = ek.cosh(X)
        elif name == "cosh":
            want = ek.sinh(X)
        elif name == "tanh":
            s = ek.rcp(ek.cosh(X)); want = s * s
        elif name == "asinh":
            want = ek.rsqrt(1.0 + X * X)
        elif name == "acosh":
            want = ek.rsqrt(X * X - 1.0)
        elif name == "atanh":
            want = ek.rcp(1.0 - X * X)
        else:
            r = ek.cbrt(X); want = 1.0 / (3.0 * (r * r))
        assert (_bits(gx) == _bits(want.numpy())).all(), name
        assert (_bits(z.numpy()) == _bits(getattr(ek, name)(X).numpy())).all()


def test_cpp_hyp_check(gpu):
    exe = os.path.join(HERE, "cpp", "hyp_check")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/hyp_check is built only where the reference headers exist")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1800)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "hyp_check ok" in r.stdout
