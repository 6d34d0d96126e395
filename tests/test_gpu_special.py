"""GPU: the Float32 operations erf, erfc, erfinv, lgamma and tgamma on an H100.  Native results against the C
restatements (tests/special_oracle.c) on the golden arguments and 2^24 random arguments per function; the same programs
on both sweep kernels, fused with other operations and reductions, at ragged sizes, in a sweep that a 64-bit value forces
onto the general kernel, and with Float16 storage; the normal-sampling step sqrt(2) * erfinv(2u - 1) against the
reference CPU path's C3 samples; FloatD gradients; and tests/cpp/special_check, which compares every Float32 input with
special.h's traced bodies on the device."""
import os
import subprocess

import numpy as np
import pytest

import special_support as ss
from test_gpu_hyperbolic import _clamp

HERE = os.path.dirname(os.path.abspath(__file__))
UNARY = ss.UNARY
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
    q = n // 4
    r[:q] = rng.uniform(-3, 3, q).astype(np.float32)
    r[q: 2 * q] = rng.uniform(-1, 1, q).astype(np.float32)
    r[2 * q: 2 * q + n // 8] = rng.uniform(-40, 40, n // 8).astype(np.float32)
    return r


def _check(name, x, got):
    """raw bits where the restatement's result is not NaN (the device's NaNs are canonical, x86 propagates payloads),
    NaN where it is NaN"""
    want = ss.unary(name, x)
    ok = ss.same_bits(got, want) & ((_bits(got) == _bits(want)) | np.isnan(want))
    assert ok.all(), (name, int((~ok).sum()), x[~ok][:5], _bits(got)[~ok][:5], _bits(want)[~ok][:5])


@pytest.mark.parametrize("name", UNARY)
def test_native_equals_restatement(ek, name):
    x = np.concatenate([np.load(os.path.join(HERE, "golden", "special.npz"))["x"], _random(51 + UNARY.index(name), 1 << 24)])
    before = int(ek.stats().fast_launches)
    got = getattr(ek, name)(ek.Float32.copy(x)).numpy()
    assert int(ek.stats().fast_launches) > before
    _check(name, x, got)


def _program(ek, a, b, c, scalar):
    """every function fused with other operations and a scalar operand"""
    t = ek.erf(a * 0.5) + ek.erfc(b) * c - ek.erfinv(ek.min_(ek.max_(a, ek.Float32(-0.99)), ek.Float32(0.99)))
    u = ek.lgamma(abs(c) + 0.5) - ek.tgamma(b * 0.5 + 2.0)
    v = ek.erf(t * scalar) + ek.erfinv(c * 0.25) * ek.erfc(scalar)
    return t + v, ek.hsum(v), ek.hmax(u)


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
        t = ((ss.unary("erf", a * f(0.5)) + ss.unary("erfc", b) * c).astype(f) - ss.unary("erfinv", _clamp(a))).astype(f)
        v = (ss.unary("erf", (t * f(0.3)).astype(f))
             + ss.unary("erfinv", (c * f(0.25)).astype(f)) * ss.unary("erfc", np.array([0.3], f))).astype(f)
        want = (t + v).astype(f)
        u = (ss.unary("lgamma", (np.abs(c) + f(0.5)).astype(f))
             - ss.unary("tgamma", ((b * f(0.5)).astype(f) + f(2)).astype(f))).astype(f)
    assert ss.same_bits(o1, want).all()
    assert ss.same_bits(m1, np.max(u))


def test_sweep_with_a_64bit_value_runs_on_the_general_kernel(ek):
    n = (1 << 20) + 7
    x = _random(61, n)
    before = int(ek.stats().fast_launches)
    X = ek.Float32.copy(x)
    wide = ek.Float64(ek.erfinv(X)) * 2.0                    # a Float64 value in the same sweep
    r = ek.erf(X) + ek.tgamma(X) - ek.erfc(X) * ek.lgamma(X)
    got_w = wide.numpy(); got_r = r.numpy()
    assert int(ek.stats().fast_launches) == before
    assert ss.same_bits((got_w / 2).astype(np.float32), ss.unary("erfinv", x)).all()
    with np.errstate(all="ignore"):
        want = (ss.unary("erf", x) + ss.unary("tgamma", x)).astype(np.float32) - (ss.unary("erfc", x) * ss.unary("lgamma", x)).astype(np.float32)
        assert ss.same_bits(got_r, want.astype(np.float32)).all()


def test_float16_storage(ek):
    n = (1 << 20) + 5
    x = np.random.default_rng(6).uniform(-4, 4, n).astype(np.float16)
    before = int(ek.stats().fast_launches)
    X = ek.Float32(ek.Float16.copy(x))
    r = ek.Float16(ek.erf(X) + ek.lgamma(X)).numpy()
    assert int(ek.stats().fast_launches) > before
    xf = x.astype(np.float32)
    want = (ss.unary("erf", xf) + ss.unary("lgamma", xf)).astype(np.float32).astype(np.float16)
    assert (r.view(np.uint16) == want.view(np.uint16)).all()


def test_normal_sampling_reproduces_the_c3_samples(ek):
    """y = sqrt(2) * erfinv(2u - 1) (the reference's tests/histogram.cpp:45) on tests/golden/c3.npz's u: the reference
    CPU path's y, bit for bit"""
    g = np.load(os.path.join(HERE, "golden", "c3.npz"))
    U = ek.Float32.copy(g["u"])
    before = int(ek.stats().fast_launches)
    y = (ek.erfinv(U * 2.0 - 1.0) * float(np.float32(np.sqrt(2.0)))).numpy()
    assert int(ek.stats().fast_launches) > before
    assert (_bits(y) == _bits(g["y"])).all()


def test_floatd_gradients_are_the_analytic_derivatives(ek):
    from scipy import special
    from enoki_b200 import autodiff as ad
    n = 4099
    rng = np.random.default_rng(10)
    F = ek.Float32
    for name in ("erf", "erfc", "erfinv"):
        lo, hi = (-0.95, 0.95) if name == "erfinv" else (-3.0, 3.0)
        xv = rng.uniform(lo, hi, n).astype(np.float32)
        x = ad.FloatD(F.copy(xv))
        ad.set_requires_gradient(x)
        z = getattr(ad, name)(x)
        ad.backward(ad.hsum(z))
        gx = ad.gradient(x).numpy()
        a = xv.astype(np.float64)
        if name == "erfinv":
            want = np.sqrt(np.pi) / 2 * np.exp(special.erfinv(a) ** 2)
        else:
            want = (1 if name == "erf" else -1) * 2 / np.sqrt(np.pi) * np.exp(-a * a)
        assert np.allclose(gx, want, rtol=1e-5, atol=0), (name, np.max(np.abs(gx - want) / np.abs(want)))
        assert (_bits(z.numpy()) == _bits(getattr(ek, name)(F.copy(xv)).numpy())).all()


def test_cpp_special_check(gpu):
    exe = os.path.join(HERE, "cpp", "special_check")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/special_check is built only where the reference headers exist")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1800)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "special_check ok" in r.stdout
