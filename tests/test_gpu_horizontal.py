"""GPU: horizontal reductions, prefix sums, stream compaction, fill and reverse against exact host references.

Every expected value is computed on the host with numpy or Python integers.  Integer results are exact with the wrap of
the result type.  Float sums and prefix sums are checked bit for bit on integer-valued data small enough that every
partial sum is exactly representable (so the result does not depend on the order the kernel folds in, and a lost carry
or a dropped tile shows up as a wrong integer), and within a derived bound on random data.  Float products use values
from {1, 2, 0.5, -1}, whose products are exact.

The reduction cases are plain builders (`reduction_cases`, `mask_cases`, `mixed_class_cases`, `many_reductions`) that
take the module and a `put(cls, array, poison)` factory; tests/test_cpu_reduction_emulator.py runs the same programs
through the planner, the assembler and the numpy interpreter of the sweep ISA."""
import contextlib
import ctypes
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TILE_PAD = 4096                 # >= the largest sweep tile (V = 16 x T = 256): a ragged last tile reads into the pad
FAST_TYPES = ("Float32", "Int32", "UInt32")     # staged 32-bit programs the fast kernel runs above 4096 elements
NARROW = ("Int8", "UInt8", "Int16", "UInt16")
TYPES32 = ("Float32", "Int32", "UInt32") + NARROW
TYPES64 = ("Float64", "Int64", "UInt64")
DTYPE = {"Float32": np.float32, "Float64": np.float64, "Int8": np.int8, "UInt8": np.uint8, "Int16": np.int16,
         "UInt16": np.uint16, "Int32": np.int32, "UInt32": np.uint32, "Int64": np.int64, "UInt64": np.uint64}
RED_SIZES = [2, 3, 31, 1023, 1024, 1025, 2047, 2048, 2049, 4095, 4096, 4097, 100_003, (1 << 22) + 5]
SCAN_SIZES = [1, 2, 7, 2047, 2048, 2049, 524_287, 524_288, 524_289, 3 * 524_288 + 5, (1 << 24) + 3]
FILL_SIZES = [1, 255, 256, 257, 270_335, 270_336, 270_337, 1_000_003]


# ------------------------------------------------------------------ exact host references
def _udt(dt):
    return np.dtype("u%d" % np.dtype(dt).itemsize)


def _wrap(v, dt):
    """Python int -> numpy scalar of integer type dt, modulo 2^width (two's complement for signed types)."""
    dt = np.dtype(dt)
    return np.array([int(v) & ((1 << (8 * dt.itemsize)) - 1)], _udt(dt)).view(dt)[0]


def int_sum(x, scale=1, shift=0):
    """sum(x * scale << shift) with the wrap of x's type (a sum modulo 2^64 reduced to the width is exact)."""
    s = int(np.sum(np.ascontiguousarray(x).view(_udt(x.dtype)), dtype=np.uint64))
    return _wrap((s * scale) << shift, x.dtype)


def int_prod(x):
    return _wrap(int(np.multiply.reduce(np.ascontiguousarray(x).view(_udt(x.dtype)).astype(np.uint64))), x.dtype)


def exact_float_sum(x, scale=1):
    """Sum of integer-valued data whose partial sums are all exact in x's type (checked here)."""
    a = np.abs(x.astype(np.float64)) * abs(scale)
    assert a.sum() < (2.0 ** 24 if x.dtype == np.float32 else 2.0 ** 53), "test data breaks the exactness bound"
    return x.dtype.type(np.sum(x.astype(np.float64) * scale))


# ------------------------------------------------------------------ test data
def integer_valued(rng, n, dt, scale=3, negative=False):
    """Integer-valued floats with scale * sum(|x|) below 2^24 (f32) / 2^53 (f64), so that the sum of x * scale is
    exact in any order.  Large n gets {-1, 0, 1} with enough zeros."""
    limit = 2 ** 24 if dt == np.float32 else 2 ** 53
    m = min((limit - 1) // (scale * n), 1 << 20)
    if m >= 1:
        x = rng.integers(-m, 0 if negative else m, n, endpoint=True)
        if negative:
            x = np.minimum(x, -1)
    else:
        q = 0.9 * limit / (scale * n)                    # density of non-zero values
        x = np.where(rng.random(n) < q, rng.choice([-1, 1], n), 0)
        if negative:
            x = -np.abs(x)
    x = x.astype(dt)
    if not negative and n >= 4:
        x[rng.integers(n)] = -0.0
        x[rng.integers(n)] = 0.0
    return x


def float_prod_data(rng, n, dt):
    """Mostly 1; up to 40 each of 2 and 0.5 and some -1: every partial product is a power of two within range."""
    x = np.ones(n, dt)
    k = min(n, 120)
    pos = rng.choice(n, size=k, replace=False)
    x[pos] = rng.choice(np.array([2.0, 0.5, -1.0], dt), size=k)
    return x


def int_data(rng, n, dt, kind):
    info = np.iinfo(dt)
    if kind == "mixed":                                  # full range with both extremes present
        x = rng.integers(info.min, info.max, n, endpoint=True, dtype=dt)
        if n >= 2:
            i, j = rng.choice(n, size=2, replace=False)
            x[i], x[j] = info.min, info.max
        return x
    if kind == "negative":                               # signed: all negative (hmax against its identity)
        return rng.integers(info.min, -1, n, endpoint=True, dtype=dt)
    if kind == "high":                                   # unsigned: all >= 2^(w-1), which a signed compare gets wrong
        return rng.integers(1 << (8 * np.dtype(dt).itemsize - 1), info.max, n, endpoint=True, dtype=dt)
    if kind == "allmax":
        return np.full(n, info.max, dt)
    if kind == "odd":                                    # products stay odd: never 0 modulo 2^w
        return rng.integers(info.min, info.max, n, endpoint=True, dtype=dt) | np.dtype(dt).type(1)
    raise ValueError(kind)


def int_poison(dt):
    """Values that would change every integer reduction if a kernel folded them in: both extremes, all-ones, 0."""
    info = np.iinfo(dt)
    return np.array([info.min, info.max, -1 if info.min < 0 else info.max, 0, 12345 % (int(info.max) + 1)], dt)


def float_poison(dt):
    return np.array([np.inf, -np.inf, 1.0e30, 0.0, -1.0e30], dt)


# ------------------------------------------------------------------ builders (shared with the CPU emulator test)
def reduction_cases(ek, put, tname, n, seed):
    """hsum / hprod / hmin / hmax over several datasets of type `tname` (n elements), plus hsum of a computed value
    whose reduction is fused into its producer.  Returns [(label, result variable, expected numpy scalar)]."""
    rng = np.random.default_rng(seed)
    T = getattr(ek, tname)
    dt = np.dtype(DTYPE[tname])
    out = []
    if dt.kind == "f":
        xs = integer_valued(rng, n, dt)
        neg = integer_valued(rng, n, dt, negative=True)
        pr = float_prod_data(rng, n, dt)
        X, N, Pr = put(T, xs, float_poison(dt)), put(T, neg, float_poison(dt)), put(T, pr, np.array([0.0, 2.0], dt))
        out += [("hsum", ek.hsum(X), exact_float_sum(xs, 1)), ("hmin", ek.hmin(X), xs.min()),
                ("hmax", ek.hmax(X), xs.max()), ("hsum(x*3)", ek.hsum(X * T(3.0)), exact_float_sum(xs, 3)),
                ("hmax(neg)", ek.hmax(N), neg.max()), ("hmin(neg)", ek.hmin(N), neg.min()),
                ("hsum(neg)", ek.hsum(N), exact_float_sum(neg, 1)),
                ("hprod", ek.hprod(Pr), dt.type(np.prod(pr.astype(np.float64))))]
        return out
    signed = dt.kind == "i"
    xs = int_data(rng, n, dt, "mixed")
    second = int_data(rng, n, dt, "negative" if signed else "high")
    odd = int_data(rng, n, dt, "odd")
    X, S, O = (put(T, a, int_poison(dt)) for a in (xs, second, odd))
    tag = "neg" if signed else "high"
    out += [("hsum", ek.hsum(X), int_sum(xs)), ("hmin", ek.hmin(X), xs.min()), ("hmax", ek.hmax(X), xs.max()),
            ("hprod", ek.hprod(X), int_prod(xs)), ("hsum(x*3)", ek.hsum(X * T(3)), int_sum(xs, 3)),
            (f"hsum({tag})", ek.hsum(S), int_sum(second)), (f"hmin({tag})", ek.hmin(S), second.min()),
            (f"hmax({tag})", ek.hmax(S), second.max()), ("hprod(odd)", ek.hprod(O), int_prod(odd))]
    if tname in ("Int32", "Int64"):
        am = int_data(rng, n, dt, "allmax")
        A = put(T, am, int_poison(dt))
        out += [("hmin(allmax)", ek.hmin(A), am.min()), ("hmax(allmax)", ek.hmax(A), am.max())]
    if tname == "UInt64":
        u = int_data(rng, n, np.uint32, "mixed")
        U = put(ek.UInt32, u, int_poison(np.uint32))
        out += [("hsum(x<<7)", ek.hsum(X << T(7)), int_sum(xs, 1, 7)),
                ("hsum(UInt64(u)<<7)", ek.hsum(ek.UInt64(U) << T(7)), _wrap(int(u.astype(np.uint64).sum()) << 7, dt))]
    return out


MASKS = ("random", "true", "false", "last", "bytes2ff", "all2ff")


def mask_cases(ek, put, n, seed, names=MASKS):
    """count / any / all over masks, including non-canonical `true` bytes (2, 0xff) of a borrowed buffer."""
    rng = np.random.default_rng(seed)
    masks = {"random": (rng.random(n) < 0.5).astype(np.uint8), "true": np.ones(n, np.uint8),
             "false": np.zeros(n, np.uint8), "last": np.zeros(n, np.uint8),
             "bytes2ff": rng.choice(np.array([0, 1, 2, 0xff], np.uint8), n),
             "all2ff": rng.choice(np.array([2, 0xff], np.uint8), n)}
    masks["last"][-1] = 1
    out = []
    for name in names:
        m = masks[name]
        M = put(ek.Mask, m, np.array([1, 0xff], np.uint8))
        c = int(np.count_nonzero(m))
        out += [(f"count({name})", ek._reduce("COUNT", M, ek.UInt32), np.uint32(c)),
                (f"any({name})", ek._reduce("ANY", M, ek.Mask), np.uint8(c > 0)),
                (f"all({name})", ek._reduce("ALL", M, ek.Mask), np.uint8(c == n))]
    return out


def mixed_class_cases(ek, put, n, seed):
    """f32 sum, i32 min, u32 max, f64 sum, i64 min, u64 max and count over the same input: one sweep, seven classes."""
    rng = np.random.default_rng(seed)
    b = integer_valued(rng, n, np.float32, scale=1).astype(np.int32)
    b[rng.integers(n)] = -7
    B = put(ek.Int32, b, int_poison(np.int32))
    u, l = b.view(np.uint32), b.astype(np.int64)
    return [("f32 hsum", ek.hsum(ek.Float32(B)), exact_float_sum(b.astype(np.float32))),
            ("i32 hmin", ek.hmin(B), b.min()),
            ("u32 hmax", ek.hmax(ek.UInt32(B)), u.max()),
            ("f64 hsum", ek.hsum(ek.Float64(B)), np.float64(l.sum())),
            ("i64 hmin", ek.hmin(ek.Int64(B)), l.min()),
            ("u64 hmax", ek.hmax(ek.UInt64(B)), l.view(np.uint64).max()),
            ("count", ek._reduce("COUNT", B > ek.Int32(0), ek.UInt32), np.uint32((b > 0).sum()))]


def many_reductions(ek, put, n, seed, k=40):
    """k > EK_MAX_RED (32) reductions recorded before one evaluation: the group must split, and all must be right."""
    rng = np.random.default_rng(seed)
    x = int_data(rng, n, np.uint32, "mixed")
    odd = int_data(rng, n, np.uint32, "odd")
    X, O = put(ek.UInt32, x, int_poison(np.uint32)), put(ek.UInt32, odd, int_poison(np.uint32))
    out = []
    for j in range(k):
        c = np.uint32(1000003 * j)
        if j % 4 == 0: out.append((f"hsum(x+{j})", ek.hsum(X + ek.UInt32(c)), int_sum(x + c)))
        elif j % 4 == 1: out.append((f"hmin(x^{j})", ek.hmin(X ^ ek.UInt32(c)), (x ^ c).min()))
        elif j % 4 == 2: out.append((f"hmax(x-{j})", ek.hmax(X - ek.UInt32(c)), (x - c).max()))
        else: out.append((f"hprod(o^{j})", ek.hprod(O ^ ek.UInt32(2 * c)), int_prod(odd ^ np.uint32(2 * c))))
    return out


def same(got, want):
    """Exact comparison of one reduction result; floats by value (so -0 == +0), integers by bits."""
    want = np.asarray(want)
    if want.dtype.kind == "f":
        return got.dtype == want.dtype and got == want
    return got.dtype.itemsize == want.dtype.itemsize and got.view(_udt(got.dtype)) == want.view(_udt(want.dtype))


def result_of(var):
    """The size-1 result of a reduction as a numpy scalar (all / any: the raw byte, which must be a canonical 0 / 1)."""
    a = var.numpy()
    return a.view(np.uint8)[0] if a.dtype == np.bool_ else a[0]


def check_cases(cases, ctx=""):
    bad = []
    for label, var, want in cases:
        got = result_of(var)
        if not same(got, want):
            bad.append(f"{label}: got {got!r}, want {want!r}")
    assert not bad, f"{ctx}: " + "; ".join(bad)


# ------------------------------------------------------------------ device staging
class Staging:
    """put(cls, array, poison): a borrowed (Type.map) variable over raw device memory, which keeps mask bytes as they
    are.  layout 'aligned': the array alone; 'ragged': followed by TILE_PAD poison elements that only a missing
    partial-tile guard would read; 'misaligned': mapped one element past a 16-byte aligned base (TMA off)."""
    def __init__(self, ek, layout="aligned"):
        self.ek, self.layout, self.bufs = ek, layout, []

    def __call__(self, cls, arr, poison):
        lib = self.ek.lib()
        arr = np.ascontiguousarray(arr)
        off = 0
        if self.layout == "ragged":
            host = np.concatenate([arr, np.resize(poison.astype(arr.dtype), TILE_PAD)])
        elif self.layout == "misaligned":
            host = np.concatenate([poison[:1].astype(arr.dtype), arr]); off = arr.itemsize
        else:
            host = arr
        p = lib.ek_malloc(host.nbytes)
        lib.ek_memcpy_to_device(p, host.ctypes.data, host.nbytes)
        self.bufs.append(p)
        return cls.map(p + off, len(arr))

    def free(self):
        lib = self.ek.lib()
        lib.ek_sync()
        for p in self.bufs:
            lib.ek_free(p)
        self.bufs = []


@contextlib.contextmanager
def kernel(ek, mode):
    """mode 'fast' / 'general': run with the fast sweep kernel allowed / disabled; 'default' leaves the setting."""
    lib = ek.lib()
    old = lib.ek_fast_mode()
    if mode != "default":
        lib.ek_set_fast_mode(1 if mode == "fast" else 0)
    try:
        yield
    finally:
        lib.ek_set_fast_mode(old)


def run_cases(ek, build, layout, mode, expect_fast, ctx):
    """Record the cases, evaluate them in one cuda_eval(), check the results and which kernel ran."""
    st = Staging(ek, layout)
    try:
        with kernel(ek, mode):
            cases = build(st)
            ek.lib().ek_stats_reset()
            ek.cuda_eval()
            fast = ek.stats().fast_launches
            check_cases(cases, ctx)
        if mode == "general":
            assert fast == 0, f"{ctx}: the fast kernel ran although it was disabled"
        elif expect_fast:
            assert fast >= 1, f"{ctx}: the fast kernel did not run"
        del cases
    finally:
        st.free()


# ------------------------------------------------------------------ reductions
# 32-bit classes (narrow types reduce in the I32 / U32 class) on both sweep kernels; 64-bit classes run on the general
# kernel only
TYPE_MODES = [(t, m) for t in TYPES32 for m in ("fast", "general")] + [(t, "default") for t in TYPES64]


@pytest.mark.parametrize("n", RED_SIZES)
@pytest.mark.parametrize("tname,mode", TYPE_MODES)
def test_reductions(gpu, tname, mode, n):
    run_cases(gpu, lambda put: reduction_cases(gpu, put, tname, n, seed=n), "aligned", mode,
              mode == "fast" and n > 4096 and tname in FAST_TYPES, f"{tname} n={n} {mode}")


@pytest.mark.parametrize("n", [31, 4097, 100_003, (1 << 22) + 5])
@pytest.mark.parametrize("layout", ["ragged", "misaligned"])
@pytest.mark.parametrize("tname,mode", TYPE_MODES)
def test_reductions_ragged_and_misaligned(gpu, tname, mode, layout, n):
    run_cases(gpu, lambda put: reduction_cases(gpu, put, tname, n, seed=7 * n), layout, mode,
              mode == "fast" and n > 4096 and tname in FAST_TYPES and layout == "ragged", f"{tname} {layout} n={n} {mode}")


@pytest.mark.parametrize("mode", ["fast", "general"])
@pytest.mark.parametrize("tname", ["Float32", "Int32"])
def test_reductions_2_24_plus_3(gpu, tname, mode):
    n = (1 << 24) + 3
    run_cases(gpu, lambda put: reduction_cases(gpu, put, tname, n, seed=3), "aligned", mode,
              mode == "fast", f"{tname} n={n} {mode}")


@pytest.mark.parametrize("mode", ["fast", "general"])
@pytest.mark.parametrize("layout", ["aligned", "ragged", "misaligned"])
@pytest.mark.parametrize("n", [2, 31, 4097, 100_003, (1 << 22) + 5])
def test_mask_reductions(gpu, n, layout, mode):
    for name in MASKS:                   # (one mask per sweep: a single 1-byte input keeps the program on the fast kernel)
        run_cases(gpu, lambda put: mask_cases(gpu, put, n, seed=n, names=(name,)), layout, mode,
                  mode == "fast" and n > 4096 and layout != "misaligned", f"mask {name} n={n} {layout} {mode}")


@pytest.mark.parametrize("n", [4097, 100_003, (1 << 22) + 5])
def test_many_classes_in_one_sweep_and_counter_reset(gpu, n):
    """Seven reduction classes in one sweep; the same program evaluated again must give the same results (the last-CTA
    tickets are back at zero after every launch)."""
    for rep in range(2):
        run_cases(gpu, lambda put: mixed_class_cases(gpu, put, n, seed=n), "aligned", "default", False,
                  f"mixed classes n={n} run {rep}")


@pytest.mark.parametrize("mode", ["fast", "general"])
@pytest.mark.parametrize("n", [31, 100_003])
def test_more_reductions_than_one_kernel_holds(gpu, n, mode):
    run_cases(gpu, lambda put: many_reductions(gpu, put, n, seed=n), "aligned", mode, mode == "fast" and n > 4096,
              f"40 reductions n={n} {mode}")


@pytest.mark.parametrize("mode", ["fast", "general"])
@pytest.mark.parametrize("n", [4097, 100_003, (1 << 22) + 5])
@pytest.mark.parametrize("tname", ["Float32", "Float64"])
def test_float_sum_rounding_bound(gpu, tname, n, mode):
    """Random non-integer data against the exact sum (math.fsum).  Every element reaches the result through at most
    d additions: c tiles folded into one register of a thread (c <= max(32, ceil(n / (132 * 128))): a sweep has at
    least 132 CTAs above 4096 elements, or one CTA of >= 128 elements per tile below), then 16 registers, 5 warp
    shuffle levels, <= 32 warps, ceil(132 * 8 / 32) = 33 CTA partials per lane of the last CTA and 5 more shuffle
    levels, so d <= c + 91 (c gets one more for a grid that does not divide the tiles evenly).  Recursive summation
    then bounds the error by gamma_d * sum|x| <= 1.01 * d * eps * sum|x| (eps = 2^-24 or 2^-53, d * eps << 1)."""
    ek = gpu
    dt = DTYPE[tname]
    rng = np.random.default_rng(n)
    x = rng.uniform(-1.0, 1.0, n).astype(dt) * dt(3.7)
    d = max(32, -(-n // (132 * 128)) + 1) + 91
    eps = 2.0 ** -24 if dt == np.float32 else 2.0 ** -53
    bound = 1.01 * d * eps * float(np.abs(x.astype(np.float64)).sum())
    st = Staging(ek)
    try:
        with kernel(ek, mode):
            r = ek.hsum(st(getattr(ek, tname), x, float_poison(dt)))
            got = float(r.numpy()[0])
        exact = math.fsum(x.astype(np.float64).tolist())
        assert abs(got - exact) <= bound, (got, exact, bound)
    finally:
        st.free()


# ------------------------------------------------------------------ raw C ABI: ek_hsum / hprod / hmin / hmax / count / all / any
def _dev(ek, host):
    lib = ek.lib()
    p = lib.ek_malloc(max(host.nbytes, 1))
    if host.nbytes:
        lib.ek_memcpy_to_device(p, host.ctypes.data, host.nbytes)
    return p


def _fetch(ek, p, dt, n=1):
    out = np.zeros(n, dt)
    if n:
        ek.lib().ek_memcpy_from_device(out.ctypes.data, p, out.nbytes)
    return out


@pytest.mark.parametrize("n", [1, 2, 4097, 100_003])
@pytest.mark.parametrize("tname", ["Float32", "Float64", "Int32", "UInt32", "Int64", "UInt64", "Int8", "UInt16"])
def test_raw_reduction_entry_points(gpu, tname, n):
    """ek_hsum / hprod / hmin / hmax return a device buffer the caller frees with ek_free (size 1 included: the Python
    mirror returns x itself there, the C ABI still reduces)."""
    ek = gpu
    L = ek.lib()
    dt = np.dtype(DTYPE[tname])
    rng = np.random.default_rng(n)
    if dt.kind == "f":
        x = integer_valued(rng, n, dt, scale=1); pr = float_prod_data(rng, n, dt)
        want = {"hsum": exact_float_sum(x), "hmin": x.min(), "hmax": x.max(), "hprod": dt.type(np.prod(pr.astype(np.float64)))}
    else:
        x = int_data(rng, n, dt, "mixed"); pr = int_data(rng, n, dt, "odd")
        want = {"hsum": int_sum(x), "hmin": x.min(), "hmax": x.max(), "hprod": int_prod(pr)}
    px, pp = _dev(ek, x), _dev(ek, pr)
    et = getattr(ek, "EK_" + tname.upper())
    try:
        for op in ("hsum", "hmin", "hmax", "hprod"):
            r = getattr(L, "ek_" + op)(et, n, pp if op == "hprod" else px)
            assert r, L.ek_last_error()
            got = _fetch(ek, r, dt)[0]
            L.ek_free(r)
            assert same(got, want[op]), (op, got, want[op])
        assert not L.ek_hsum(et, 0, px) and L.ek_last_error()
    finally:
        L.ek_free(px); L.ek_free(pp)


@pytest.mark.parametrize("n", [1, 31, 4097, 100_003])
def test_raw_count_all_any(gpu, n):
    ek = gpu
    L = ek.lib()
    rng = np.random.default_rng(n)
    for m in (rng.choice(np.array([0, 1, 2, 0xff], np.uint8), n), rng.choice(np.array([2, 0xff], np.uint8), n),
              np.zeros(n, np.uint8), (rng.random(n) < 0.01).astype(np.uint8) * 2):
        p = _dev(ek, m)
        try:
            c = int(np.count_nonzero(m))
            assert L.ek_count(n, p) == c
            assert L.ek_all(n, p) == int(c == n)
            assert L.ek_any(n, p) == int(c > 0)
        finally:
            L.ek_free(p)


# ------------------------------------------------------------------ ek_psum
PSUM_TYPES = ["Int32", "UInt32", "Int64", "UInt64", "Float32", "Float64"]


def psum_data(rng, n, tname):
    dt = np.dtype(DTYPE[tname])
    if dt.kind == "f":
        return integer_valued(rng, n, dt, scale=1)
    if dt == np.uint32:                                  # large values: the prefix wraps many times
        return int_data(rng, n, dt, "high")
    return int_data(rng, n, dt, "mixed")


def psum_want(x):
    if x.dtype.kind == "f":
        return np.cumsum(x.astype(np.float64)).astype(x.dtype)    # every prefix is exact (checked in integer_valued)
    u = _udt(x.dtype)
    return np.cumsum(x.view(u), dtype=u).view(x.dtype)            # numpy's unsigned cumsum wraps like the kernel


def run_psum(ek, tname, x, layout):
    L = ek.lib()
    dt = x.dtype
    poison = float_poison(dt) if dt.kind == "f" else int_poison(dt)
    st = Staging(ek, layout)
    try:
        v = st(getattr(ek, tname), x, poison)
        p = L.ek_psum(getattr(ek, "EK_" + tname.upper()), len(x), L.ek_var_ptr(v.index))
        assert p, L.ek_last_error()
        got = _fetch(ek, p, dt, len(x))
        L.ek_free(p)
        del v
    finally:
        st.free()
    return got


@pytest.mark.parametrize("n", SCAN_SIZES)
@pytest.mark.parametrize("tname", PSUM_TYPES)
def test_psum_exact(gpu, tname, n):
    """Integer prefixes exact with wrap (uint32 wraps), float prefixes bit-exact on integer-valued data.  Above 524 288
    elements (256 tiles of 2048) the tile totals are scanned in several rounds; 2^24 + 3 is 8193 tiles, 33 rounds."""
    x = psum_data(np.random.default_rng(n), n, tname)
    got, want = run_psum(gpu, tname, x, "aligned"), psum_want(x)
    bad = np.flatnonzero(got.view(_udt(got.dtype)) != want.view(_udt(want.dtype)))
    assert bad.size == 0, f"{bad.size} wrong prefixes, first at {bad[0]}: got {got[bad[0]]!r}, want {want[bad[0]]!r}"


@pytest.mark.parametrize("n", [2049, 524_289, 3 * 524_288 + 5])
@pytest.mark.parametrize("layout", ["ragged", "misaligned"])
@pytest.mark.parametrize("tname", PSUM_TYPES)
def test_psum_ragged_and_misaligned(gpu, tname, layout, n):
    x = psum_data(np.random.default_rng(n + 1), n, tname)
    got, want = run_psum(gpu, tname, x, layout), psum_want(x)
    assert (got.view(_udt(got.dtype)) == want.view(_udt(want.dtype))).all()


@pytest.mark.parametrize("n", [2049, 524_289, 3 * 524_288 + 5])
@pytest.mark.parametrize("tname", ["Float32", "Float64"])
def test_psum_rounding_bound(gpu, tname, n):
    """Random non-integer data (multiples of 2^-20, so the exact prefixes are int64 cumsums).  Prefix i is the tile's
    offset plus the scan inside the tile; its value passes through at most d roundings: 8 serial items and 5 + 3
    shuffle levels to form each tile total, the same again plus one subtraction (inclusive - own) inside the tile scan,
    8 levels and one subtraction in the scan of one round of 256 tile totals, and one carry addition per earlier round:
    d <= 64 + rounds (rounds = ceil(tiles / 256)).  The subtractions take partial sums that include the rest of i's
    tile, so the error bound is 1.01 * d * eps * A_i with A_i = sum of |x_j| up to the end of i's 2048-element tile."""
    dt = DTYPE[tname]
    rng = np.random.default_rng(n)
    q = np.rint(rng.uniform(-5.3, 5.3, n) * 2.0 ** 20).astype(np.int64)
    x = (q * 2.0 ** -20).astype(dt)                       # exact in f32 too: |q| < 2^24
    got = run_psum(gpu, tname, x, "aligned").astype(np.float64)
    exact = np.cumsum(q).astype(np.float64) * 2.0 ** -20   # (one rounding to f64, far inside the bound)
    tiles = -(-n // 2048)
    rounds = -(-tiles // 256)
    eps = 2.0 ** -24 if dt == np.float32 else 2.0 ** -53
    cum = np.cumsum(np.abs(x.astype(np.float64)))
    tile_end = np.minimum((np.arange(n) // 2048 + 1) * 2048, n) - 1
    bound = 1.01 * (64 + rounds) * eps * cum[tile_end]
    err = np.abs(got - exact)
    assert (err <= bound).all(), (int(np.argmax(err / bound)), float((err / bound).max()))


def test_psum_abi_edges(gpu):
    ek = gpu
    L = ek.lib()
    p = _dev(ek, np.arange(8, dtype=np.int8))
    try:
        assert not L.ek_psum(ek.EK_UINT32, 0, p) and L.ek_last_error()
        assert not L.ek_psum(ek.EK_INT8, 8, p) and L.ek_last_error()
    finally:
        L.ek_free(p)


# ------------------------------------------------------------------ ek_compress
COMPRESS_TYPES = {1: "UInt8", 2: "Int16", 4: "Float32", 8: "UInt64"}


def compress_masks(rng, n):
    m = {"false": np.zeros(n, np.uint8), "true": np.ones(n, np.uint8),
         "alternating": (np.arange(n) % 2).astype(np.uint8), "first": np.zeros(n, np.uint8), "last": np.zeros(n, np.uint8)}
    m["first"][0] = 1
    m["last"][-1] = 1
    for dens in (0.01, 0.5, 0.99):
        m[f"random{dens}"] = (rng.random(n) < dens).astype(np.uint8)
    m["bytes2ff"] = rng.choice(np.array([0, 2, 0xff], np.uint8), n)
    return m


@pytest.mark.parametrize("n", SCAN_SIZES)
@pytest.mark.parametrize("es", [1, 2, 4, 8])
def test_compress_exact(gpu, es, n):
    ek = gpu
    L = ek.lib()
    rng = np.random.default_rng(n * 10 + es)
    data = rng.integers(0, 256, n * es, dtype=np.uint8).view(_udt(np.dtype("u%d" % es)))
    et = getattr(ek, "EK_" + COMPRESS_TYPES[es].upper())
    pd = _dev(ek, data)
    try:
        for name, m in compress_masks(rng, n).items():
            pm = _dev(ek, m)
            od, osz = ctypes.c_void_p(), ctypes.c_size_t()
            try:
                assert L.ek_compress(et, n, pd, pm, ctypes.byref(od), ctypes.byref(osz)) == 0, L.ek_last_error()
                want = data[m != 0]
                assert osz.value == want.size, (name, osz.value, want.size)
                assert od.value, name                      # a real (freeable) buffer even when nothing was selected
                got = _fetch(ek, od.value, data.dtype, osz.value)
                L.ek_free(od.value)
                assert (got == want).all(), (name, int(np.flatnonzero(got != want)[0]))
            finally:
                L.ek_free(pm)
        od, osz = ctypes.c_void_p(1), ctypes.c_size_t(7)
        assert L.ek_compress(et, 0, pd, pd, ctypes.byref(od), ctypes.byref(osz)) == 0 and osz.value == 0
    finally:
        L.ek_free(pd)


# ------------------------------------------------------------------ ek_fill / ek_reverse
GUARD = 37                       # sentinel elements on each side


def _guarded(ek, n, es, seed):
    """A device buffer of GUARD + n + GUARD elements pre-filled with random sentinel bytes; returns (ptr, host copy)."""
    host = np.random.default_rng(seed).integers(0, 256, (n + 2 * GUARD) * es, dtype=np.uint8)
    return _dev(ek, host), host


@pytest.mark.parametrize("n", FILL_SIZES)
@pytest.mark.parametrize("es", [1, 2, 4, 8])
def test_fill(gpu, es, n):
    """Non-zero 2-, 4- and 8-byte values run the fill kernel (a grid-stride loop above 132 * 8 * 256 = 270 336
    elements); 1-byte values and zero use cudaMemsetAsync."""
    ek = gpu
    L = ek.lib()
    for value in (0x8877665544332211 & ((1 << (8 * es)) - 1), 0):
        p, host = _guarded(ek, n, es, n + es)
        try:
            L.ek_fill(p + GUARD * es, es, value, n)
            got = _fetch(ek, p, np.uint8, host.size)
        finally:
            L.ek_free(p)
        want = host.copy()
        want[GUARD * es:(GUARD + n) * es] = np.frombuffer(value.to_bytes(8, "little")[:es] * n, np.uint8)
        assert (got == want).all(), (hex(value), int(np.flatnonzero(got != want)[0]) // es - GUARD)


@pytest.mark.parametrize("n", FILL_SIZES)
@pytest.mark.parametrize("es", [1, 2, 4, 8])
def test_reverse(gpu, es, n):
    ek = gpu
    L = ek.lib()
    src = np.random.default_rng(n).integers(0, 256, n * es, dtype=np.uint8)
    ps = _dev(ek, src)
    p, host = _guarded(ek, n, es, n + 3)
    try:
        L.ek_reverse(p + GUARD * es, ps, es, n)
        got = _fetch(ek, p, np.uint8, host.size)
    finally:
        L.ek_free(p); L.ek_free(ps)
    want = host.copy()
    want[GUARD * es:(GUARD + n) * es] = src.reshape(n, es)[::-1].reshape(-1)
    assert (got == want).all(), int(np.flatnonzero(got != want)[0]) // es - GUARD


# ------------------------------------------------------------------ tape psum / reverse edges at multi-round size
@pytest.mark.parametrize("tname", ["Float32", "Float64"])
def test_tape_psum_and_reverse_edges(gpu, tname):
    """The psum edge's adjoint is reverse(psum(reverse(g))) -- the suffix sum of g -- and the reverse edge's is g[::-1],
    at 3 * 524 288 + 5 elements (several rounds of tile totals in the scan)."""
    ek = gpu
    L = ek.lib()
    T = getattr(ek, tname)
    et = getattr(ek, "EK_" + tname.upper())
    dt = DTYPE[tname]
    n = 3 * 524_288 + 5
    g = integer_valued(np.random.default_rng(5), n, dt, scale=1)     # sum|g| < 2^24: every suffix sum is exact
    want = np.cumsum(g[::-1].astype(np.float64))[::-1].astype(dt)

    def gradient(node_kind, seed):
        leaf = L.ek_tape_append_leaf(et, n)
        node = (L.ek_tape_append_psum if node_kind == "psum" else L.ek_tape_append_reverse)(et, leaf)
        assert leaf and node, L.ek_last_error()
        if seed is None:
            assert L.ek_tape_backward(et, node, 1) == 0, L.ek_last_error()
        else:
            G = T.copy(seed)
            assert L.ek_tape_set_gradient(et, node, G.index, 1) == 0, L.ek_last_error()
            del G
            assert L.ek_tape_backward_static(et, 1) == 0, L.ek_last_error()
        h = L.ek_tape_gradient(et, leaf)
        assert h
        L.ek_inc_ref_ext(h)
        got = T.from_index(h).numpy()
        L.ek_tape_dec_ref_ext(et, node); L.ek_tape_dec_ref_ext(et, leaf)
        assert L.ek_tape_node_count(et) == 0
        return got

    got = gradient("psum", g)
    assert (got.view(_udt(got.dtype)) == want.view(_udt(want.dtype))).all(), int(np.flatnonzero(got != want)[0])
    got = gradient("psum", None)
    assert (got == (n - np.arange(n)).astype(dt)).all()
    got = gradient("reverse", g)
    assert (got.view(_udt(got.dtype)) == g[::-1].view(_udt(g.dtype))).all()
