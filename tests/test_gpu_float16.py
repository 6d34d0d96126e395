"""GPU: Float16 arrays as a storage format on the H100.  Conversions of every binary16 bit pattern and of every rounding
boundary against the reference's half (tests/golden/convert_f16.npz) and numpy, data movement (copies, literals, select,
bit casts, gather, scatter, compaction), C2 with Float16 storage on both sweep kernels, and the PyTorch float16 interop."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "convert_f16.npz")
ALL_HALVES = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)


@pytest.fixture()
def fast_mode(ek, gpu):
    yield
    ek.lib().ek_set_fast_mode(1)


def _bits(a):
    return np.ascontiguousarray(a).view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


@pytest.mark.parametrize("target", ["Float32", "Float64", "Int8", "UInt8", "Int16", "UInt16", "Int32", "UInt32", "Int64",
                                    "UInt64"])
def test_every_half_bit_pattern_to(ek, gpu, target):
    gold = np.load(GOLD)
    h = ek.Float16.copy(ALL_HALVES.view(np.float16))
    got = getattr(ek, target)(h).numpy()
    want = gold[f"half_{target}_0"]
    f = ALL_HALVES.view(np.float16).astype(np.float32)
    nan = np.isnan(f)
    if target.startswith("Float"):
        assert (_bits(got)[~nan] == _bits(want)[~nan]).all()
        assert (_bits(f.astype(got.dtype))[~nan] == _bits(got)[~nan]).all()        # exact widening
        assert np.isnan(got[nan]).all()
        if target == "Float32":      # the H100's cvt.f32.f16 returns the canonical NaN; F16C keeps sign and payload
            assert (_bits(got)[nan] == 0x7fffffff).all()
    else:
        # Float16 -> integer is Float16 -> Float32 and then the Float32 rules of DESIGN.md 4, for inf and NaN as well
        via_f32 = getattr(ek, target)(ek.Float32.copy(f)).numpy()
        assert (got == via_f32).all()
        fin = np.isfinite(f)
        assert (got[fin] == want[fin]).all()


@pytest.mark.parametrize("mode", [1, 2])
def test_floor2int_and_ceil2int_from_every_half(ek, gpu, mode):
    gold = np.load(GOLD)
    h = ek.Float16.copy(ALL_HALVES.view(np.float16))
    got = (ek.floor2int if mode == 1 else ek.ceil2int)(ek.Int32, h).numpy()
    f = ALL_HALVES.view(np.float16).astype(np.float32)
    fin = np.isfinite(f)
    want = (np.floor if mode == 1 else np.ceil)(f[fin]).astype(np.int32)
    assert (got[fin] == want).all() and (got[fin] == gold[f"half_Int32_{mode}"][fin]).all()
    assert (got[~fin] == np.int32(-2 ** 31)).all()


def _nan_check(x, got):
    """NaN in gives NaN out.  The H100's cvt.rn.f16.f32 returns the canonical NaN 0x7fff for every NaN; F16C
    (the reference) keeps the sign and the top payload bits instead, so the NaN bits are compared with 0x7fff."""
    nan = np.isnan(x)
    assert np.isnan(got.view(np.float16)[nan]).all()
    assert (got[nan] == 0x7fff).all(), sorted({hex(v) for v in got[nan]})[:8]
    return nan


def _rounding_boundaries():
    """Float32 bit patterns around every rounding boundary of binary16, both signs: each midpoint between neighbouring
    halves and the floats just below / above it, every half, the overflow threshold 65520, the subnormal range and its
    lower end 2^-25, zeros, infinities and NaNs (the golden file holds the same set for every 7th half)."""
    h = np.arange(0x7c00, dtype=np.uint32)
    lo = h.astype(np.uint16).view(np.float16).astype(np.float32).view(np.uint32).astype(np.uint64)
    hi = (h + 1).astype(np.uint16).view(np.float16).astype(np.float32).view(np.uint32).astype(np.uint64)
    mid = (lo + hi) // 2
    extra = [0x477fe000, 0x477fefff, 0x477ff000, 0x477ff001, 0x7f7fffff, 0x7f800000, 0x00000001, 0x00800000, 0x32ffffff,
             0x33000000, 0x33000001, 0x33800000, 0x387fc000, 0x387fe000, 0x38800000, 0x7f800001, 0x7fc00000, 0x7fffffff]
    v = np.concatenate([mid - 1, mid, mid + 1, lo, np.array(extra, np.uint64)]).astype(np.uint32)
    return np.concatenate([v, v | np.uint32(0x80000000)]).view(np.float32)


def test_float32_to_float16_on_every_rounding_boundary(ek, gpu):
    gold = np.load(GOLD)
    x = gold["x_Float32"]
    got = ek.Float16(ek.Float32.copy(x)).numpy().view(np.uint16)
    nan = _nan_check(x, got)
    assert (got[~nan] == gold["Float32_half"][~nan]).all()
    # every boundary: numpy's float16 rounds to nearest even as well
    xb = _rounding_boundaries()
    gb = ek.Float16(ek.Float32.copy(xb)).numpy().view(np.uint16)
    nb = _nan_check(xb, gb)
    with np.errstate(over="ignore"):
        assert (gb[~nb] == xb[~nb].astype(np.float16).view(np.uint16)).all()


def test_float32_to_float16_on_random_bit_patterns(ek, gpu):
    bits = np.random.default_rng(24).integers(0, 1 << 32, 1 << 24, dtype=np.uint64).astype(np.uint32)
    x = bits.view(np.float32)
    got = ek.Float16(ek.Float32.copy(x)).numpy().view(np.uint16)
    nan = _nan_check(x, got)
    with np.errstate(over="ignore"):
        want = x.astype(np.float16).view(np.uint16)
    bad = (got != want) & ~nan
    assert not bad.any(), (int(bad.sum()), bits[bad][:4], got[bad][:4], want[bad][:4])


@pytest.mark.parametrize("src", ["Float64", "Int8", "UInt8", "Int16", "UInt16", "Int32", "UInt32", "Int64", "UInt64"])
def test_other_types_to_float16_go_through_float32(ek, gpu, src):
    gold = np.load(GOLD)
    x = gold[f"x_{src}"]
    got = ek.Float16(getattr(ek, src).copy(x)).numpy().view(np.uint16)
    want = gold[f"{src}_half"]
    nan = np.isnan(x) if src == "Float64" else np.zeros(len(x), bool)
    assert (got[~nan] == want[~nan]).all(), (x[got != want][:4], got[got != want][:4], want[got != want][:4])
    with np.errstate(over="ignore"):
        assert (got[~nan] == x[~nan].astype(np.float32).astype(np.float16).view(np.uint16)).all()
    if src == "Float64":
        assert np.isnan(got.view(np.float16)[nan]).all()


def test_float64_double_rounding(ek, gpu):
    x = np.array([1 + 2.0 ** -11 + 2.0 ** -30] * 5000, np.float64)
    got = ek.Float16(ek.Float64.copy(x)).numpy().view(np.uint16)
    assert (got == 0x3C00).all()                 # a single rounding (cvt.rn.f16.f64) would give 0x3c01
    assert ek.Float16(1 + 2.0 ** -11 + 2.0 ** -30).coeff(0).view(np.uint16) == 0x3C00


def test_copies_literals_and_fetch_element(ek, gpu):
    h = ALL_HALVES.view(np.float16)
    a = ek.Float16.copy(h)
    assert (a.numpy().view(np.uint16) == ALL_HALVES).all()                 # NaN payloads included: only bits move
    assert a.coeff(0x3C00).view(np.uint16) == 0x3C00 and a.coeff(0xFE01).view(np.uint16) == 0xFE01
    full = ek.Float16.full(np.float16(-2.5), 4097).numpy()
    assert (full.view(np.uint16) == np.float16(-2.5).view(np.uint16)).all() and full.size == 4097
    lit = ek.select(ek.Mask.copy(np.arange(1 << 16) % 2 == 0), ek.Float16(0.1), a)   # literal inside a wide sweep
    got = lit.numpy().view(np.uint16)
    assert (got[0::2] == np.float16(np.float32(0.1)).view(np.uint16)).all()


def test_select_and_bitcasts(ek, gpu):
    rng = np.random.default_rng(3)
    n = 100_003
    a = rng.integers(0, 1 << 16, n).astype(np.uint16)
    b = rng.integers(0, 1 << 16, n).astype(np.uint16)
    m = rng.integers(0, 2, n).astype(np.bool_)
    fa, fb = ek.Float16.copy(a.view(np.float16)), ek.Float16.copy(b.view(np.float16))
    assert (ek.select(ek.Mask.copy(m), fa, fb).numpy().view(np.uint16) == np.where(m, a, b)).all()
    assert (ek.reinterpret(ek.UInt16, fa).numpy() == a).all()
    assert (ek.reinterpret(ek.Int16, fa).numpy() == a.view(np.int16)).all()
    assert (ek.Int32(ek.reinterpret(ek.Int16, fa)).numpy() == a.view(np.int16).astype(np.int32)).all()
    back = ek.reinterpret(ek.Float16, ek.Int16.copy(b.view(np.int16)))
    assert (back.numpy().view(np.uint16) == b).all()
    assert (ek.Float32(back).numpy().view(np.uint32)[~np.isnan(b.view(np.float16))] ==
            b.view(np.float16).astype(np.float32).view(np.uint32)[~np.isnan(b.view(np.float16))]).all()


def _gather(ek, cls, source, index, mask, stride):
    """enoki_b200.gather with an explicit stride in bytes (a field of a struct of Float16 values)."""
    L = ek.lib()
    assert L.ek_set_scatter_gather_operand(source.index, 1) == 0
    try:
        ptr = L.ek_var_register_ptr(L.ek_var_ptr(source.index))
        try:
            return cls.from_index(ek._append(cls.Type, "GATHER", ptr, index.index, mask.index, stride))
        finally:
            L.ek_dec_ref_ext(ptr)
    finally:
        L.ek_set_scatter_gather_operand(0, 0)


def test_gathers(ek, gpu):
    rng = np.random.default_rng(5)
    table = rng.integers(0, 1 << 16, 3000).astype(np.uint16)
    n = 50_001
    idx = rng.integers(0, 3000, n).astype(np.uint32)
    m = rng.random(n) < 0.8
    t = ek.Float16.copy(table.view(np.float16))
    g = ek.gather(ek.Float16, t, ek.UInt32.copy(idx), ek.Mask.copy(m)).numpy().view(np.uint16)
    assert (g == np.where(m, table[idx], 0)).all()
    # stride 4: the second half of (half, half) pairs
    pairs = rng.integers(0, 1 << 16, 2 * 3000).astype(np.uint16)
    tp = ek.Float16.copy(pairs.view(np.float16))
    gs = _gather(ek, ek.Float16, tp, ek.UInt32.copy(idx), ek.Mask(True), 4).numpy().view(np.uint16)
    # the base pointer of element k is 4k bytes in: the first half of pair k
    assert (gs == pairs[2 * idx]).all()
    # a small Float32 table staged in shared memory, read into a Float16 output
    ft = rng.uniform(-3, 3, 1000).astype(np.float32)
    i2 = rng.integers(0, 1000, n).astype(np.uint32)
    f = ek.Float32.copy(ft)
    before = ek.stats().launches
    h = ek.Float16(ek.gather(ek.Float32, f, ek.UInt32.copy(i2)))
    prog = ek.debug_program()
    assert any("GATHER_32_SMEM" in [prog["ops"][t_[0]] for t_ in sw["body"]] for sw in prog["sweeps"])
    assert (h.numpy().view(np.uint16) == ft[i2].astype(np.float16).view(np.uint16)).all()
    assert ek.stats().launches > before


def test_masked_scatter(ek, gpu):
    rng = np.random.default_rng(6)
    n = 40_000
    target = rng.integers(0, 1 << 16, n).astype(np.uint16)
    perm = rng.permutation(n).astype(np.uint32)
    vals = rng.integers(0, 1 << 16, n).astype(np.uint16)
    m = rng.random(n) < 0.5
    t = ek.Float16.copy(target.view(np.float16))
    ek.scatter(t, ek.Float16.copy(vals.view(np.float16)), ek.UInt32.copy(perm), ek.Mask.copy(m))
    want = target.copy()
    want[perm[m]] = vals[m]
    assert (t.numpy().view(np.uint16) == want).all()


def test_compress_fill_reverse(ek, gpu):
    L = ek.lib()
    rng = np.random.default_rng(7)
    n = 70_001
    a = rng.integers(0, 1 << 16, n).astype(np.uint16)
    m = rng.random(n) < 0.3
    fa, fm = ek.Float16.copy(a.view(np.float16)), ek.Mask.copy(m)
    out, size = ctypes.c_void_p(), ctypes.c_size_t()
    assert L.ek_compress(ek.EK_FLOAT16, n, fa.data(), fm.data(), ctypes.byref(out), ctypes.byref(size)) == 0
    c = ek.Float16.map(out.value, size.value, True)
    assert size.value == int(m.sum()) and (c.numpy().view(np.uint16) == a[m]).all()
    r = ek.Float16.empty(n)
    L.ek_reverse(r.data(), fa.data(), 2, n)
    assert (r.numpy().view(np.uint16) == a[::-1]).all()
    L.ek_fill(r.data(), 2, 0xBC00, n)
    assert (r.numpy().view(np.uint16) == 0xBC00).all()


def test_psum_refuses_float16(ek, gpu):
    a = ek.Float16.copy(np.ones(100, np.float16))
    assert not ek.lib().ek_psum(ek.EK_FLOAT16, 100, a.data())
    assert "Float16" in ek.lib().ek_last_error().decode()


def _c2_ref(oracle, P, xs):
    f = [np.ascontiguousarray(x.astype(np.float32)) for x in xs]
    want = np.zeros(len(f[0]), np.float32)
    oracle.or_c2(P(f[0]), P(f[1]), P(f[2]), P(f[3]), P(want), ctypes.c_size_t(len(want)))
    return want.astype(np.float16)


def _c2(ek, hs):
    x0, x1, x2, x3 = (ek.Float32(h) for h in hs)
    t = ek.fmadd(x0, x1, x2)
    return ek.Float16(ek.fmadd(ek.sin(ek.fmadd(x3, ek.exp(-(t * t)), x0)), x1, ek.sqrt(abs(t))))


@pytest.mark.parametrize("n,offset", [(1, 0), (31, 0), (4095, 0), (4097, 0), ((1 << 20) + 3, 0), ((1 << 20) + 3, 1),
                                      (1 << 26, 0)])
def test_c2_with_float16_storage_on_both_kernels(ek, gpu, fast_mode, oracle, P, n, offset):
    rng = np.random.default_rng(n + offset)
    xs = [rng.uniform(-4, 4, n).astype(np.float16) for _ in range(4)]
    owners = [ek.Float16.copy(np.concatenate([np.zeros(offset, np.float16), x])) for x in xs]
    # offset = 1: the inputs start one element (2 bytes) into their allocation, which rules out the TMA bulk copy
    hs = [ek.Float16.map(o.data() + 2 * offset, n) for o in owners] if offset else owners
    want = _c2_ref(oracle, P, xs)
    outs = {}
    for fast in (0, 1):
        ek.lib().ek_set_fast_mode(fast)
        before = int(ek.stats().fast_launches)
        got = _c2(ek, hs).numpy()
        used_fast = int(ek.stats().fast_launches) - before
        if fast == 0 or n <= 4096:
            assert used_fast == 0
        else:
            assert used_fast > 0, "Float16-storage C2 did not run on the fast kernel"
        outs[fast] = got.view(np.uint16)
        bad = outs[fast] != want.view(np.uint16)
        assert not bad.any(), (fast, int(bad.sum()), got[bad][:4], want[bad][:4])
    assert (outs[0] == outs[1]).all()


def test_torch_float16_round_trip(ek, gpu):
    torch = pytest.importorskip("torch")
    import enoki_b200.torch_interop  # noqa: F401
    h = ALL_HALVES.view(np.float16)
    a = ek.Float16.copy(h)
    t = a.torch()
    assert t.dtype == torch.float16 and t.is_cuda
    assert (t.cpu().numpy().view(np.uint16) == ALL_HALVES).all()
    back = ek.Float16.from_torch(t * 2)
    want = (torch.from_numpy(h.copy()).cuda() * 2).cpu().numpy().view(np.uint16)
    assert (back.numpy().view(np.uint16) == want).all()
    src = torch.linspace(-3, 3, 1001, device="cuda", dtype=torch.float32)
    f = ek.Float16.from_torch(src)                   # converted to float16 by torch first
    assert (f.numpy().view(np.uint16) == src.cpu().numpy().astype(np.float16).view(np.uint16)).all()


def test_cpp_half_check(gpu):
    exe = os.path.join(HERE, "cpp", "half_check")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/half_check is built only where the reference headers exist")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "half_check ok" in r.stdout
