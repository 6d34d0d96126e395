"""GPU: the Float32 Carlson integrals carlson_rf, carlson_rd and carlson_rc on an H100.  Native results against the C
restatements (tests/ell_oracle.c), bit for bit, on both sweep kernels (the kernel asserted through the launch counters),
at ragged sizes, with literal and computed operands in every position and with Float16 storage around them; against the
reference CPU path's golden vectors (tests/golden/ell.npz) within the measured ulp bound of DESIGN.md 4; the Python API,
comp_ellint_1 / comp_ellint_2 among it; and tests/cpp/ell_check, which compares the native operations with special.h's
traced bodies on the device."""
import os
import subprocess

import numpy as np
import pytest

import ell_support as es

HERE = os.path.dirname(os.path.abspath(__file__))
pytestmark = pytest.mark.gpu
# the largest distance to the reference CPU path on arguments within 2^-60 ... 2^60: every body takes rcp(mu), which is
# correctly rounded here and rcpps + one Newton step there
ULP_BOUND = {"carlson_rf": 2, "carlson_rd": 2, "carlson_rc": 2, "comp_ellint_1": 3, "comp_ellint_2": 4}


@pytest.fixture(autouse=True)
def fast_mode(ek, gpu):
    yield
    ek.lib().ek_set_fast_mode(1)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _check(got, want, what):
    ok = es.same_bits(got, want)
    assert ok.all(), (what, int((~ok).sum()), _bits(got)[~ok][:5], _bits(want)[~ok][:5])


def _ulp(a, b):
    ai, bi = (np.asarray(v, np.float32).view(np.int32).astype(np.int64) for v in (a, b))
    ai = np.where(ai < 0, -(ai & 0x7fffffff), ai)
    bi = np.where(bi < 0, -(bi & 0x7fffffff), bi)
    return np.abs(ai - bi)


def _args(seed, n, arity):
    """random bit patterns, then valid arguments over 2^-40 ... 2^40 (x = 0 for some)"""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 1 << 32, (arity, n), dtype=np.uint64).astype(np.uint32).view(np.float32)
    h = n // 2
    a[:, h:] = np.exp2(rng.uniform(-40, 40, (arity, n - h))).astype(np.float32)
    a[0, h::10] = 0
    return list(a)


def _call(ek, name, *args):
    return getattr(ek, name)(*args)


@pytest.mark.parametrize("fast", [1, 0])
@pytest.mark.parametrize("name", es.TERNARY + es.BINARY)
def test_native_equals_restatement(ek, name, fast):
    ek.lib().ek_set_fast_mode(fast)
    arity = 3 if name in es.TERNARY else 2
    for n in (1 << 20, 4097, 31):
        args = _args(91 + n, n, arity)
        before = ek.stats()
        got = _call(ek, name, *(ek.Float32.copy(a) for a in args)).numpy()
        after = ek.stats()
        assert int(after.sweep_launches) == int(before.sweep_launches) + 1
        # (sweeps of at most 4096 elements run on the general kernel)
        want_fast = fast if n > 4096 else 0
        assert int(after.fast_launches) - int(before.fast_launches) == want_fast, "the sweep ran on the wrong kernel"
        _check(got, es.call(name, *args), (name, n, fast))


@pytest.mark.parametrize("name", es.TERNARY + es.BINARY)
def test_against_the_reference_cpu_path(ek, name):
    d = np.load(os.path.join(HERE, "golden", "ell.npz"))
    args = (d["tx"], d["ty"], d["tz"]) if name in es.TERNARY else (d["px"], d["py"])
    got = _call(ek, name, *(ek.Float32.copy(a) for a in args)).numpy()
    _check(got, es.call(name, *args), name)
    ok = lambda a: (a == 0) | ((a >= 2.0 ** -60) & (a <= 2.0 ** 60))
    m = np.logical_and.reduce([ok(a) for a in args])
    g, w = got[m], d[name][m]
    assert (np.isnan(g) == np.isnan(w)).all() and (np.isinf(g) == np.isinf(w)).all()
    assert (np.signbit(g) == np.signbit(w)).all()
    assert _ulp(g, w).max() <= ULP_BOUND[name], (name, int(_ulp(g, w).max()))


def _complete(k):
    """comp_ellint_1 / 2 composed from the restatements as special.h composes them"""
    f = np.float32
    k2 = (k * k).astype(f)
    y = (f(1) - k2).astype(f)
    rf, rd = es.call("carlson_rf", 0, y, 1), es.call("carlson_rd", 0, y, 1)
    return {"comp_ellint_1": rf, "comp_ellint_2": (rf - (f(1.0 / 3.0) * k2).astype(f) * rd).astype(f)}


def test_complete_integrals(ek):
    """the golden k (4008 elements: the general kernel) against the restatements and the reference CPU path, then the
    same k repeated past 4096 elements, where the sweep runs on the fast kernel with x = 0 and z = 1 broadcast from the
    uniform pool (FF_BU / FF_CU)"""
    d = np.load(os.path.join(HERE, "golden", "ell.npz"))
    k = d["k"]
    for name, w in _complete(k).items():
        before = int(ek.stats().sweep_launches)
        got = getattr(ek, name)(ek.Float32.copy(k)).numpy()
        assert int(ek.stats().sweep_launches) == before + 1, "not one sweep"
        _check(got, w, name)
        assert _ulp(got, d[name]).max() <= ULP_BOUND[name], (name, int(_ulp(got, d[name]).max()))
    kl = np.tile(k, 5)
    assert len(kl) > 4096
    for name, w in _complete(kl).items():
        before = ek.stats()
        got = getattr(ek, name)(ek.Float32.copy(kl)).numpy()
        after = ek.stats()
        assert int(after.sweep_launches) == int(before.sweep_launches) + 1, "not one sweep"
        assert int(after.fast_launches) == int(before.fast_launches) + 1, "the sweep did not run on the fast kernel"
        _check(got, w, name + " (fast kernel)")


@pytest.mark.parametrize("fast", [1, 0])
def test_fused_programs_with_literals_and_float16_storage(ek, fast):
    """literal operands in every position (uniform operands of the frame), computed y / z (x loaded by the instruction),
    the reversed carlson_rc, and Float16 inputs and outputs around them, in one sweep"""
    ek.lib().ek_set_fast_mode(fast)
    rng = np.random.default_rng(5)
    n = 100_003
    a, b, c = (rng.uniform(0.01, 4, n).astype(np.float32) for _ in range(3))
    h = rng.uniform(0.01, 4, n).astype(np.float16)
    A, B, C = (ek.Float32.copy(v) for v in (a, b, c))
    H = ek.Float32(ek.Float16.copy(h))
    f = np.float32
    with np.errstate(all="ignore"):
        b2, c3, h32 = (b * f(2)).astype(f), (c * f(3)).astype(f), h.astype(f)
    before = ek.stats()
    r1 = ek.carlson_rf(A, B * 2.0, C * 3.0)
    r2 = ek.carlson_rd(1.5, B, A)
    r3 = ek.carlson_rc(A, B * 2.0)
    r4 = ek.carlson_rc(0.5, H)
    r5 = ek.Float16(ek.carlson_rf(H, 1.0, C) + ek.carlson_rd(A, 2.0, 3.0))
    got = [r.numpy() for r in (r1, r2, r3, r4)] + [r5.numpy()]
    after = ek.stats()
    assert int(after.sweep_launches) == int(before.sweep_launches) + 1
    assert int(after.fast_launches) - int(before.fast_launches) == fast
    _check(got[0], es.call("carlson_rf", a, b2, c3), "rf")
    _check(got[1], es.call("carlson_rd", 1.5, b, a), "rd")
    _check(got[2], es.call("carlson_rc", a, b2), "rc")
    _check(got[3], es.call("carlson_rc", 0.5, h32), "rc literal x")
    want5 = (es.call("carlson_rf", h32, 1.0, c) + es.call("carlson_rd", a, 2.0, 3.0)).astype(f).astype(np.float16)
    assert (got[4].view(np.uint16) == want5.view(np.uint16)).all()


def test_cpp_ell_check(gpu):
    exe = os.path.join(HERE, "cpp", "ell_check")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/ell_check is built only where the reference headers exist")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1800)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ell_check ok" in r.stdout
