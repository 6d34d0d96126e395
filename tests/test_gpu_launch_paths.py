"""GPU: the launch paths the host chooses before a sweep runs, each asserted and then checked against exact references.

Before every launch `cuda_eval()` decides how the program, its literals and its inputs reach the kernel (kernel
parameters, a shared-memory copy or global memory; TMA staging or direct loads), which kernel configuration runs, and
whether a group that does not fit one kernel is split.  Most of these paths only run for unusual programs, and an
interpreter that takes a wrong one still returns plausible numbers.  Every case here therefore

1. asserts the path from the dry-run plan (`debug_program()`), the launch line of log level 1 (`V=, T=, stages=,
   grid=`) or `stats().fast_launches`, so that a case that stops reaching its path fails instead of passing vacuously;
2. evaluates on the GPU;
3. compares bit for bit (NaN == NaN) with a host reference: numpy float32 / float64 add, sub and mul are correctly
   rounded, integer arithmetic wraps, and every float sum is over integer values whose partial sums are exact.

The builders take the module and a `put(cls, array)` factory; tests/test_cpu_launch_paths.py runs the same builders on
fake device addresses and checks the planned path (and, where the numpy interpreter of the sweep ISA supports every
operation, the values) without a GPU."""
import contextlib
import gc
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

INLINE_PROG = 448               # instructions carried in the kernel parameters (EK_INLINE_PROG)
SMEM_PROG = 24 * 1024 // 16     # a longer program is copied to shared memory up to 24 KB of instructions
LIT_INLINE = 128                # literal words carried in the kernel parameters (EK_MAX_LIT_INLINE)
STAGE_UNITS = 8                 # slot units of TMA-staged inputs (EK_STAGE_UNIT_BUDGET); the rest are direct loads
MAX_SCALAR = 64                 # size-1 evaluated inputs per kernel (EK_MAX_SCALAR)
TILE_PAD = 4096                 # elements, >= the largest tile (fast kernel: 16 x 256): a load that ignored the ragged
                                # last tile's bound would still stay inside the allocation

# choose_config's candidates (V, T, stages, CTAs per SM); the small list serves sweeps of at most 4096 elements
WIDE = [(8, 256, 1, 4), (8, 256, 1, 3), (8, 256, 2, 2), (8, 256, 1, 2), (8, 256, 2, 1), (8, 256, 1, 1),
        (8, 128, 2, 1), (8, 128, 1, 1),
        (4, 128, 2, 1), (4, 64, 2, 1), (4, 32, 2, 1)]
SMALL = [(4, 32, 2, 1), (4, 128, 2, 1), (8, 256, 2, 1)]


# ------------------------------------------------------------------ model of choose_config (general kernel)
def smem_need(sw, V, T, stages):
    """Shared memory of a general-kernel launch of sweep `sw` (a debug_program() entry), as smem_layout() lays it out."""
    n_uni = len(sw["lits"]) + len(sw["argw"]) + 2 * len(sw["scalars"])
    n_prog = len(sw["init"]) + len(sw["body"]) + len(sw["fini"])
    n_in = sum(2 if es == 8 else 1 for _v, _u, es in sw["staged"])
    off = n_uni * 16 + 8 * 8 + 33 * 8
    off = (off + 15) & ~15
    if n_prog * 16 <= SMEM_PROG * 16:
        off += n_prog * 16
    off += extra_bytes(sw)
    off = (off + 1023) & ~1023
    return off + T * V * 4 * (sw["n_tmp"] + (stages if n_in else 2) * n_in)


def extra_bytes(sw):
    return 0          # (no case here uses shared-memory tables or bins)


def general_config(sw, n, optin=227 * 1024):
    """(V, T, stages, CTAs per SM) the general kernel runs sweep `sw` of n elements with, or None."""
    per_sm = 228 * 1024 - 1024
    n_in = sum(2 if es == 8 else 1 for _v, _u, es in sw["staged"])
    if n <= 4096:
        pick = 0 if n <= 128 else 1 if n <= 512 else 2
        for V, T, st, c in SMALL[pick:]:
            if smem_need(sw, V, T, 2) <= optin:
                return (V, T, 2, 1)
    for V, T, st, c in WIDE:
        st = st if n_in else 2
        need = smem_need(sw, V, T, st)
        if need <= optin and (need + 1024) * c <= per_sm + 1024:
            return (V, T, st, c)
    return None


def prog_len(sw):
    return len(sw["init"]) + len(sw["body"]) + len(sw["fini"])


def fast_len(sw):
    f = sw.get("fast")
    return None if f is None else len(f["init"]) + len(f["body"]) + len(f["fini"])


def ops(prog, sw):
    return [prog["ops"][i[0]] for sec in ("init", "body", "fini") for i in sw[sec]]


# ------------------------------------------------------------------ device data
class Device:
    """put(cls, array): a borrowed (Type.map) variable over raw device memory followed by TILE_PAD poison elements.
    misaligned=True maps it one element past a 16-byte aligned base (TMA staging is then off for the whole sweep).
    The memory is returned by the `clean` fixture once the test has dropped its variables (Device.release)."""
    live = []

    def __init__(self, ek, misaligned=False):
        self.ek, self.misaligned, self.bufs = ek, misaligned, []
        Device.live.append(self)

    def __call__(self, cls, arr, misaligned=None):
        lib = self.ek.lib()
        arr = np.ascontiguousarray(arr)
        mis = self.misaligned if misaligned is None else misaligned
        pad = np.full(TILE_PAD * arr.itemsize, 0x5b, np.uint8).view(arr.dtype)
        host = np.concatenate([pad[:1], arr, pad]) if mis else np.concatenate([arr, pad])
        p = lib.ek_malloc(host.nbytes)
        lib.ek_memcpy_to_device(p, host.ctypes.data, host.nbytes)
        self.bufs.append(p)
        return cls.map(p + (arr.itemsize if mis else 0), len(arr))

    @staticmethod
    def release(ek):
        lib = ek.lib()
        lib.ek_sync()
        for d in Device.live:
            for p in d.bufs:
                lib.ek_free(p)
        Device.live = []


def same_bits(got, want):
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype == np.bool_ or want.dtype == np.bool_:
        return (got.astype(np.bool_) == want.astype(np.bool_)).all()
    w = np.broadcast_to(want.astype(got.dtype), got.shape)
    u = np.dtype("u%d" % got.dtype.itemsize)
    ok = got.view(u) == np.ascontiguousarray(w).view(u)
    if got.dtype.kind == "f":
        ok |= np.isnan(got) & np.isnan(w)
    return ok.all()


def check(cases, ctx=""):
    bad = []
    for label, var, want in cases:
        got = var.numpy()
        if not same_bits(got, want):
            w = np.broadcast_to(np.asarray(want).astype(got.dtype), got.shape)
            diff = np.flatnonzero(got != w)
            bad.append(f"{label}: {len(diff)} elements differ, first at {diff[:3]}: got {got[diff[:3]]}, want {w[diff[:3]]}")
    assert not bad, f"{ctx}: " + "; ".join(bad)


@contextlib.contextmanager
def fast_mode(ek, on):
    lib = ek.lib()
    lib.ek_set_fast_mode(1 if on else 0)
    try:
        yield
    finally:
        lib.ek_set_fast_mode(1)


LAUNCH = re.compile(r"ek_eval\(\): launching sweep \(n=(\d+), in=\d+, out=\d+, ops=\d+, slots=(\d+), V=(\d+), T=(\d+), "
                    r"stages=(\d+), grid=(\d+), smem=(\d+)\)")


def evaluate(ek, capfd):
    """cuda_eval() with the launch lines logged: [(n, slots, V, T, stages, grid, smem)] in launch order, and the
    number of sweeps that ran on the fast kernel."""
    capfd.readouterr()
    lib = ek.lib()
    lib.ek_stats_reset()
    lib.ek_set_log_level(1)
    try:
        ek.cuda_eval()
    finally:
        lib.ek_set_log_level(0)
    err = capfd.readouterr().err
    return [tuple(int(g) for g in m.groups()) for m in LAUNCH.finditer(err)], ek.stats().fast_launches


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------ builders
def chain(ek, x, xn, length, cls):
    """`length` dependent arithmetic instructions on x: alternately y = c - y and y = y + d with small integer
    literals, so that every intermediate is an integer and exact in float32 / float64."""
    dt = xn.dtype
    y, yn = x, xn.copy()
    for k in range(length):
        c = float(k % 7 + 1)
        if k % 2 == 0:
            y = c - y; yn = dt.type(c) - yn
        else:
            y = y + c; yn = yn + dt.type(c)
    return y, yn


def reduce_raw(ek, op, x):
    """A reduction node even for a size-1 operand (hsum() etc. return a size-1 operand itself)."""
    return type(x).from_index(ek._append(x.Type, op, x.index))


def delivery_case(ek, put, n, length, tname="Float64", seed=0):
    """A chain of `length` instructions over one input, kept, plus its maximum: a fused reduction gives the program an
    init and a fini section.  Returns cases."""
    rng = np.random.default_rng(seed)
    cls = getattr(ek, tname)
    xn = rng.integers(-1000, 1000, n).astype(np.float64 if tname == "Float64" else np.float32)
    x = put(cls, xn)
    y, yn = chain(ek, x, xn, length, cls)
    m = reduce_raw(ek, "HMAX", y)
    return [("chain", y, yn), ("hmax(chain)", m, yn.max())]


def tuned(ek, build, target, measure, start):
    """Record build(length) with `length` tuned so that measure(debug_program()) == target; every step adds one
    instruction, so this converges in a few rounds.  Returns (cases, program)."""
    length = start
    for _ in range(6):
        cases = build(length)
        prog = ek.debug_program()
        got = measure(prog)
        if got == target:
            return cases, prog
        del cases
        gc.collect()
        length += target - got if got is not None else -8
    raise AssertionError(f"could not tune the program to {target} instructions (last {got})")


def literal_case(ek, put, n, n_words, seed=0, base=0):
    """x plus a run of distinct literals (alternating sign): the program's literal pool holds `n_words` words."""
    rng = np.random.default_rng(seed)
    xn = rng.integers(-1000, 1000, n).astype(np.float32)
    y, yn = put(ek.Float32, xn), xn.copy()
    for k in range(n_words):
        c = float((base + k + 1) * (-1) ** k)
        y = y + c; yn = yn + np.float32(c)
    return [("literals", y, yn)]


def evict_program(ek, y, yn, i):
    """Program i of the cache-eviction sequence: 128 literal words shared by all programs and one of its own."""
    for k in range(LIT_INLINE):
        c = float((k + 1) * (-1) ** k)
        y = y + c; yn = yn + np.float32(c)
    return y - float(i + 1000), yn - np.float32(i + 1000)


def straddle_case(ek, put, n, seed=0):
    """127 distinct 32-bit literals and then one 64-bit literal: its two words sit at pool words 127 and 128."""
    rng = np.random.default_rng(seed)
    xn = rng.integers(-1000, 1000, n).astype(np.float32)
    y, yn = put(ek.Float32, xn), xn.copy()
    for k in range(127):
        c = float(k + 1000)
        y = y + c; yn = yn + np.float32(c)
    big = np.float64(1.0) + np.float64(2.0) ** -40            # distinct halves: 0x3ff00000 00001000... both matter
    z = ek.Float64(y) + ek.Float64(float(big))
    return [("f32 part", y, yn), ("f64 with pair literal", z, yn.astype(np.float64) + big)]


def live_temps_case(ek, put, n, k_temps, n_inputs=1, n_extra_lits=0, seed=0, tname="Float32"):
    """t_i = x_(i mod n_inputs) + i for i < k_temps, used once by a left-to-right sum and once more by a reversed
    difference: every t_i is live across the program, so it needs about k_temps slots.  n_extra_lits distinct literals
    go into the pool through one more chain.  Integer data: every value is exact."""
    rng = np.random.default_rng(seed)
    cls = getattr(ek, tname)
    dt = np.dtype(np.float32 if tname == "Float32" else np.float64)
    xs_n = [rng.integers(-100, 100, n).astype(dt) for _ in range(n_inputs)]
    xs = [put(cls, a) for a in xs_n]
    t = [xs[i % n_inputs] + float(i + 1) for i in range(k_temps)]
    tn = [xs_n[i % n_inputs] + dt.type(i + 1) for i in range(k_temps)]
    a, an = t[0], tn[0]
    for i in range(1, k_temps):
        a = a + t[i]; an = an + tn[i]
    b, bn = t[-1], tn[-1]
    for i in range(k_temps - 2, -1, -1):
        b = b - t[i]; bn = bn - tn[i]
    out, outn = a * 3.0 + b, an * dt.type(3) + bn
    cases = [("live temps", out, outn)]
    if n_extra_lits:
        e, en = xs[0], xs_n[0].copy()
        for k in range(n_extra_lits):
            c = float(100_000 + k)
            e = e - c if k % 2 else e + c
            en = en - dt.type(c) if k % 2 else en + dt.type(c)
        cases.append(("literal pool", e, en))
    return cases


def pressure_case(ek, put, n, k_temps=500, seed=0):
    """The sum and the reversed difference of t_i = x + i as two kept results: together every t_i is live across the
    kernel (more slots than any configuration holds); each result alone uses every t_i once."""
    rng = np.random.default_rng(seed)
    xn = rng.integers(-100, 100, n).astype(np.float32)
    x = put(ek.Float32, xn)
    t = [x + float(i + 1) for i in range(k_temps)]
    tn = [xn + np.float32(i + 1) for i in range(k_temps)]
    a, an = t[0], tn[0]
    for i in range(1, k_temps):
        a = a + t[i]; an = an + tn[i]
    b, bn = t[-1], tn[-1]
    for i in range(k_temps - 2, -1, -1):
        b = b - t[i]; bn = bn - tn[i]
    return [("sum", a, an), ("difference", b, bn)]


DIRECT_NARROW = {                 # type: data covering the sign bits and the extremes
    "Int8": np.array([-128, 127, -1, 0, 1, -2], np.int8),
    "UInt8": np.array([0, 255, 128, 127, 1, 0x80], np.uint8),
    "Int16": np.array([-0x8000, 0x7fff, -1, 0, 1, -2], np.int16),
    "UInt16": np.array([0x8000, 0xffff, 0, 1, 0x7fff, 2], np.uint16),
    "Int64": np.array([-2 ** 63, 2 ** 63 - 1, -1, 0, 1, -(2 ** 32)], np.int64),
    "UInt64": np.array([2 ** 63, 2 ** 64 - 1, 0, 1, 2 ** 32, 2 ** 63 - 1], np.uint64),
    "Mask": np.array([0, 1, 2, 0xff, 0, 1], np.uint8),
}


def direct_f32_case(ek, put, n, n_inputs=17, seed=0):
    """A sum of n_inputs Float32 arrays: 8 are staged, the rest are LDG_32 direct loads (every add correctly rounded)."""
    rng = np.random.default_rng(seed)
    xs_n = [rng.standard_normal(n).astype(np.float32) for _ in range(n_inputs)]
    xs = [put(ek.Float32, a) for a in xs_n]
    s, sn = xs[0], xs_n[0]
    for x, xn in zip(xs[1:], xs_n[1:]):
        s = s + x; sn = sn + xn
    return [("sum of inputs", s, sn)]


def direct_f64_case(ek, put, n, n_inputs=5, seed=0):
    """n_inputs Float64 arrays: 4 fill the 8 staging units, the fifth is an LDG_64 direct load."""
    rng = np.random.default_rng(seed)
    xs_n = [rng.standard_normal(n) for _ in range(n_inputs)]
    xs = [put(ek.Float64, a) for a in xs_n]
    s, sn = xs[0], xs_n[0]
    for x, xn in zip(xs[1:], xs_n[1:]):
        s = s * x + x; sn = sn * xn + xn
    return [("f64 inputs", s, sn)]


def direct_narrow_case(ek, put, n, seed=0):
    """Eight Float32 inputs fill the staging budget first; then one direct input each of Int8, UInt8, Int16, UInt16,
    Int64, UInt64 and Mask, carried to an output by a widening conversion, an xor or a select."""
    rng = np.random.default_rng(seed)
    fs_n = [rng.standard_normal(n).astype(np.float32) for _ in range(STAGE_UNITS)]
    fs = [put(ek.Float32, a) for a in fs_n]
    s, sn = fs[0], fs_n[0]
    for x, xn in zip(fs[1:], fs_n[1:]):
        s = s + x; sn = sn + xn
    cases = [("staged sum", s, sn)]
    for tname, pattern in DIRECT_NARROW.items():
        data = np.resize(pattern, n)
        rng.shuffle(data[len(pattern):])
        x = put(getattr(ek, tname), data)
        if tname in ("Int8", "Int16"):
            cases.append((tname, ek.Int32(x), data.astype(np.int32)))
        elif tname in ("UInt8", "UInt16"):
            cases.append((tname, ek.UInt32(x), data.astype(np.uint32)))
        elif tname == "Int64":
            k = np.int64(0x5555aaaa33cc0ff0)
            cases.append((tname, x ^ ek.Int64(int(k)), data ^ k))
        elif tname == "UInt64":
            k = np.uint64(0xa5a5f00f0ff01234)
            cases.append((tname, x ^ ek.UInt64(int(k)), data ^ k))
        else:
            cases.append((tname, ek.select(x, ek.Int32(1), ek.Int32(7)), np.where(data != 0, 1, 7).astype(np.int32)))
    return cases


def staged_mixed_case(ek, put, n, misaligned=(True, True, True, True), seed=0):
    """Staged Int8, Int16, UInt16 and Int64 inputs (3 + 2 units) widened or carried into outputs: on a misaligned
    input the tiles are loaded by plain stores and unpacked from those bytes."""
    rng = np.random.default_rng(seed)
    a = rng.integers(-128, 128, n).astype(np.int8)
    b = rng.integers(-0x8000, 0x8000, n).astype(np.int16)
    c = rng.integers(0, 0x10000, n).astype(np.uint16)
    d = rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64)
    A, B, C, D = (put(cls, v, misaligned=m) for cls, v, m in
                  zip((ek.Int8, ek.Int16, ek.UInt16, ek.Int64), (a, b, c, d), misaligned))
    s = ek.Int32(A) + ek.Int32(B) * 3 + ek.Int32(ek.UInt32(C))
    sn = a.astype(np.int32) + b.astype(np.int32) * np.int32(3) + c.astype(np.int32)
    k = np.int64(0x0123456789abcdef)
    return [("narrow sum", s, sn), ("int64", D ^ ek.Int64(int(k)), d ^ k)]


def many_outputs_case(ek, put, n, count=300, seed=77):
    """`count` kept results over 6 inputs with a shared fmadd: more output pointers than one kernel's argument words
    hold, so the group is split and the shared sub-expression recomputed."""
    rng = np.random.default_rng(seed)
    xs_n = [rng.integers(-64, 64, n).astype(np.float32) for _ in range(6)]
    X = [put(ek.Float32, a) for a in xs_n]
    base = ek.fmadd(X[0], X[1], X[2])
    base_n = xs_n[0] * xs_n[1] + xs_n[2]           # integers below 2^13: exact, the same as a fused multiply-add
    cases = []
    for k in range(count):
        e = (base + X[k % 6]) * float(k + 1) - X[(k + 3) % 6]
        cases.append((f"out{k}", e, (base_n + xs_n[k % 6]) * np.float32(k + 1) - xs_n[(k + 3) % 6]))
    return cases


SCALAR_TYPES = ("Float32", "Int32", "Int8", "Int16", "UInt8", "UInt16", "Mask")


NARROW_SCALAR_TYPES = {1, 2, 3, 4, 12}      # EK_INT8, EK_UINT8, EK_INT16, EK_UINT16, EK_BOOL (include/enoki_b200.h)


def scalar_values(tname, k):
    """The k-th scalar of type tname: the extremes and a small negative value, Mask bytes 0, 1, 2 and 0xff."""
    if tname == "Mask":
        return np.array([[0, 1, 2, 0xff][k % 4]], np.uint8)
    if tname == "Float32":
        return np.array([float(k) - 40.0], np.float32)
    if tname == "Int32":
        return np.array([-k * 1001], np.int32)
    dt = np.dtype(tname.lower())
    info = np.iinfo(dt)
    return np.array([[info.min, info.max, -3 if info.min < 0 else 3][k % 3]], dt)


def scalar_case(ek, put, n, count=100, groups=4, seed=3):
    """`count` distinct evaluated size-1 inputs of mixed types (negative Int8 / Int16, Mask bytes 2 and 0xff), every one
    read by a wide operation: a Mask scalar selects between two wide values, any other scalar is picked by a wide mask
    and then widened to Int32 (exact: a carrier, no narrow arithmetic).  `groups` wide results share the scalars out, so
    that their group holds all `count` and is split when that is more than one kernel takes."""
    rng = np.random.default_rng(seed)
    xn = rng.integers(-50, 50, n).astype(np.int32)
    x = put(ek.Int32, xn)
    cases = []
    k = 0
    for g, chunk in enumerate(np.array_split(np.arange(count), groups)):
        acc, accn = x, xn.copy()
        for _ in chunk:
            tname = SCALAR_TYPES[k % len(SCALAR_TYPES)]
            v = scalar_values(tname, k)
            s = put(getattr(ek, tname), v)
            if tname == "Mask":
                acc = acc + ek.select(s, x, x + 1)
                accn = accn + (xn if v[0] else xn + np.int32(1))
            else:
                c = k % 7 - 3
                T = getattr(ek, tname)
                acc = acc + ek.Int32(ek.select(x > c, s, T(0)))
                accn = accn + np.where(xn > c, v.astype(np.int64)[0], 0).astype(np.int32)
            k += 1
        cases.append((f"group{g}", acc, accn))
    return cases


def check_scalar_plan(prog, n, count):
    """Every scalar is read by a wide sweep of n elements, the narrow and Mask types among them, and the wide group is
    split so that no kernel takes more than MAX_SCALAR."""
    sweeps = prog["sweeps"]
    assert all(s["n"] == n for s in sweeps), [s["n"] for s in sweeps]
    assert len(sweeps) >= 2 and all(len(s["scalars"]) <= MAX_SCALAR for s in sweeps), [len(s["scalars"]) for s in sweeps]
    assert sum(len(s["scalars"]) for s in sweeps) == count
    assert NARROW_SCALAR_TYPES <= {t for s in sweeps for _v, t in s["scalars"]}


def scatter_split_case(ek, put, n, count=240, seed=5):
    """A group that must split and carries side effects: `count` plain scatters into one target, every one at the same
    permuted index (so each element is written by one thread, in recording order: the last scatter must win), integer
    scatter_adds into a second target, and `count` kept outputs that overflow one kernel's argument words."""
    rng = np.random.default_rng(seed)
    perm = rng.permutation(n).astype(np.uint32)
    xn = rng.integers(-100, 100, n).astype(np.float32)
    x = put(ek.Float32, xn)
    idx = put(ek.UInt32, perm)
    target = put(ek.Float32, np.full(n, -7.0, np.float32))
    hist = put(ek.UInt32, np.zeros(n, np.uint32))
    tn = np.full(n, -7.0, np.float32)
    hn = np.zeros(n, np.uint32)
    cases = []
    for k in range(count):
        if k % 2 == 0:
            v = x + float(k)
            ek.scatter(target, v, idx, x > float(k - count // 2))
            m = xn > np.float32(k - count // 2)
            tn[perm[m]] = (xn + np.float32(k))[m]
        else:
            ek.scatter_add(hist, ek.UInt32(k), idx)
            hn[perm] += np.uint32(k)
        o = x * float(k + 1)
        cases.append((f"out{k}", o, xn * np.float32(k + 1)))
    cases += [("scatter target", target, tn), ("scatter_add target", hist, hn)]
    return cases


def split_reduction_case(ek, put, n, count=300, seed=9):
    """A split group whose first half holds a reduction that a later phase consumes."""
    rng = np.random.default_rng(seed)
    xn = rng.integers(-8, 8, n).astype(np.float32)
    x = put(ek.Float32, xn)
    s = ek.hsum(x * 2.0)
    sn = np.float32(np.sum(xn.astype(np.float64) * 2))
    cases = [(f"out{k}", x + float(k), xn + np.float32(k)) for k in range(count)]
    cases.append(("consumer of the reduction", x * 4.0 - s, xn * np.float32(4) - sn))
    return cases


# ------------------------------------------------------------------ tests
@pytest.fixture()
def clean(gpu):
    """Starts from an empty trace; afterwards (the test's variables are gone by then) returns the device memory."""
    gc.collect()
    gpu.cuda_eval()
    gpu.lib().ek_sync()
    yield gpu
    gc.collect()
    Device.release(gpu)


def run(ek, capfd, cases, ctx):
    lines, fast = evaluate(ek, capfd)
    check(cases, ctx)
    return lines, fast


# A. program delivery
@pytest.mark.parametrize("n", [1, 4096, 4097, (1 << 21) + 3])
@pytest.mark.parametrize("target", [INLINE_PROG, INLINE_PROG + 1, SMEM_PROG, SMEM_PROG + 1, 4000])
@pytest.mark.parametrize("tname", ["Float64", "Float32"])
def test_program_delivery(clean, capfd, tname, target, n):
    ek = clean
    put = Device(ek)
    with fast_mode(ek, False):
        cases, prog = tuned(ek, lambda L: delivery_case(ek, put, n, L, tname), target,
                            lambda p: prog_len(p["sweeps"][0]) if len(p["sweeps"]) == 1 else None, target - 4)
        sw = prog["sweeps"][0]
        if n > 1:
            assert sw["init"] and sw["fini"], "the program has no init / fini section"
        lines, fast = run(ek, capfd, cases, f"{tname} {target} instructions, n={n}")
    assert len(lines) == 1 and fast == 0


@pytest.mark.parametrize("target", [INLINE_PROG, INLINE_PROG + 1])
def test_fast_kernel_program_length(clean, capfd, target):
    """The fast kernel takes a lowered program of up to 448 instructions; one more and the general kernel runs it."""
    ek = clean
    put = Device(ek)
    n = 3 * 4096 + 5

    cases, prog = fast_tuned(ek, put, n, target)
    lines, fast = run(ek, capfd, cases, f"fast kernel, {target} lowered instructions")
    assert len(lines) == 1 and fast == (1 if target == INLINE_PROG else 0)


def fast_tuned(ek, put, n, target):
    """The delivery chain with a lowered fast-kernel program of `target` instructions.  Above 448 the dry run no longer
    offers a lowering, so 449 is 448 plus one chain instruction (each lowers to exactly one instruction)."""
    holder = {}

    def build(L):
        holder["L"] = L
        return delivery_case(ek, put, n, L, "Float32")
    cases, prog = tuned(ek, build, INLINE_PROG, lambda p: fast_len(p["sweeps"][0]), INLINE_PROG - 8)
    if target == INLINE_PROG:
        return cases, prog
    general = prog_len(prog["sweeps"][0])
    del cases
    gc.collect()
    cases = build(holder["L"] + target - INLINE_PROG)
    prog = ek.debug_program()
    assert prog_len(prog["sweeps"][0]) == general + target - INLINE_PROG
    assert fast_len(prog["sweeps"][0]) is None, "a lowered program longer than 448 instructions was offered"
    return cases, prog


# B. literal pools
@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("words", [LIT_INLINE - 1, LIT_INLINE, LIT_INLINE + 1, LIT_INLINE + 2, 3300])
def test_literal_pool(clean, capfd, words, fast):
    ek = clean
    put = Device(ek)
    n = 5 * 4096 + 3
    with fast_mode(ek, fast):
        cases, prog = tuned(ek, lambda k: literal_case(ek, put, n, k), words,
                            lambda p: len(p["sweeps"][0]["lits"]), words)
        expect_fast = fast and fast_len(prog["sweeps"][0]) is not None
        lines, nfast = run(ek, capfd, cases, f"{words} literal words")
    assert nfast == (1 if expect_fast else 0)
    if fast and words <= LIT_INLINE + 2:
        assert nfast == 1, "the 32-bit literal program did not run on the fast kernel"
    if words == 3300:                          # 48 KB of uniform pool pushes the configuration below 4 CTAs / SM
        want = general_config(prog["sweeps"][0], n)
        assert want[3] < 4 and lines[0][2:5] == want[:3], (want, lines)


def test_literal_pair_straddles_the_inline_limit(clean, capfd):
    ek = clean
    put = Device(ek)
    cases = straddle_case(ek, put, 70_001)
    sw = ek.debug_program()["sweeps"]
    lits = [s for s in sw if len(s["lits"]) == LIT_INLINE + 1]
    assert lits, [len(s["lits"]) for s in sw]
    pair = (np.uint64(lits[0]["lits"][LIT_INLINE]) << np.uint64(32)) | np.uint64(lits[0]["lits"][LIT_INLINE - 1])
    assert pair == np.float64(1.0 + 2.0 ** -40).view(np.uint64)
    run(ek, capfd, cases, "64-bit literal at words 127/128")


def test_uniform_pool_overflow_splits_or_refuses(clean, capfd):
    """More than 4096 uniform words: two results split into two kernels; a single result is refused, and nothing runs."""
    ek = clean
    put = Device(ek)
    n = 10_007
    cases = literal_case(ek, put, n, 2200, seed=1) + literal_case(ek, put, n, 2200, seed=2, base=5000)
    assert [len(s["lits"]) for s in ek.debug_program()["sweeps"]] == [2200, 2200]
    lines, _ = run(ek, capfd, cases, "two chains of 2200 literals")
    assert len(lines) == 2
    put = Device(ek)
    rng = np.random.default_rng(4)
    xn = rng.integers(-9, 9, n).astype(np.float32)
    y = put(ek.Float32, xn)
    for k in range(4200):
        y = y + float(k + 10_000)
    before = ek.stats().launches
    with pytest.raises(ek.EnokiError, match="uniform pool overflow|split"):
        ek.cuda_eval()
    assert ek.stats().launches == before
    del y


# C. program cache
def cache_program(ek, put, xn, lit_shift=0, n_lits=LIT_INLINE + 2):
    y, yn = put(ek.Float32, xn), xn.copy()
    for k in range(n_lits):
        c = float((k + 1 + (lit_shift if k == n_lits - 1 else 0)) * (-1) ** k)
        y = y + c; yn = yn + np.float32(c)
    return y, yn


@pytest.mark.parametrize("fast", [False, True])
def test_program_cache_hit_and_miss(clean, capfd, fast):
    ek = clean
    n = 20_011
    rng = np.random.default_rng(1)
    with fast_mode(ek, fast):
        for shift in (0, 0, 1000, 0):          # same program with new data (hit), one literal changed (miss), back
            put = Device(ek)
            xn = rng.integers(-500, 500, n).astype(np.float32)
            y, yn = cache_program(ek, put, xn, shift)
            sw = ek.debug_program()["sweeps"][0]
            assert len(sw["lits"]) > LIT_INLINE and sw["config"]["inline_lit"] == 0, "the literals do not go through the cache"
            assert sw["config"]["fast"] == int(fast)
            _lines, nfast = run(ek, capfd, [("cached program", y, yn)], f"literal shift {shift}")
            assert nfast == int(fast)
            del y


def test_program_cache_eviction(clean, capfd):
    """300 distinct programs whose literals live in device memory, each consuming the previous one's output without a
    synchronisation in between: the cache is emptied at least once while earlier sweeps are still running."""
    ek = clean
    n = 50_003
    put = Device(ek)
    rng = np.random.default_rng(2)
    xn = rng.integers(-100, 100, n).astype(np.float32)
    y, yn = put(ek.Float32, xn), xn.copy()
    keep = []
    for i in range(300):
        y, yn = evict_program(ek, y, yn, i)
        if i == 0:
            assert len(ek.debug_program()["sweeps"][0]["lits"]) == LIT_INLINE + 1
        ek.cuda_eval()
        keep.append((f"program {i}", y, yn))
    first, firstn = evict_program(ek, put(ek.Float32, xn), xn, 0)
    keep.append(("first program again", first, firstn))
    run(ek, capfd, keep, "cache eviction")


# D. direct loads
@pytest.mark.parametrize("misaligned", [False, True])
@pytest.mark.parametrize("fast", [False, True])
def test_direct_loads_f32(clean, capfd, fast, misaligned):
    ek = clean
    put = Device(ek, misaligned)
    n = 3 * 4096 * 16 + 1001
    with fast_mode(ek, fast):
        cases = direct_f32_case(ek, put, n)
        prog = ek.debug_program()
        sw = prog["sweeps"][0]
        assert ops(prog, sw).count("LDG_32") == 9 and len(sw["staged"]) == STAGE_UNITS
        _lines, nfast = run(ek, capfd, cases, "17 Float32 inputs")
    assert nfast == (1 if fast else 0)


@pytest.mark.parametrize("misaligned", [False, True])
def test_direct_loads_f64(clean, capfd, misaligned):
    ek = clean
    put = Device(ek, misaligned)
    cases = direct_f64_case(ek, put, 3 * 2048 * 132 + 77)
    prog = ek.debug_program()
    sw = prog["sweeps"][0]
    assert ops(prog, sw).count("LDG_64") == 1 and len(sw["staged"]) == 4
    run(ek, capfd, cases, "5 Float64 inputs")


@pytest.mark.parametrize("misaligned", [False, True])
@pytest.mark.parametrize("n", [4097, 3 * 2048 * 132 + 13])
def test_direct_loads_narrow(clean, capfd, n, misaligned):
    ek = clean
    put = Device(ek, misaligned)
    cases = direct_narrow_case(ek, put, n)
    prog = ek.debug_program()
    sw = prog["sweeps"][0]
    o = ops(prog, sw)
    for op in ("LDG_S8", "LDG_U8", "LDG_S16", "LDG_U16", "LDG_64"):
        assert op in o, (op, o)
    assert o.count("LDG_U8") == 2 and o.count("LDG_64") == 2
    run(ek, capfd, cases, "direct narrow / 64-bit inputs")


# E. misaligned staged inputs
@pytest.mark.parametrize("which", ["all", "int8 only", "int64 only", "none"])
def test_misaligned_staged_inputs(clean, capfd, which):
    ek = clean
    put = Device(ek)
    mis = {"all": (True,) * 4, "int8 only": (True, False, False, False), "int64 only": (False, False, False, True),
           "none": (False,) * 4}[which]
    n = 4 * 2048 * 132 * 4 + 999                 # >= 3 tiles per CTA at any configuration of 8 elements per thread
    cases = staged_mixed_case(ek, put, n, mis)
    prog = ek.debug_program()
    sw = prog["sweeps"][0]
    assert sorted(es for _v, _u, es in sw["staged"]) == [1, 2, 2, 8] and "LDG" not in " ".join(ops(prog, sw))
    lines, _ = run(ek, capfd, cases, f"misaligned staged inputs ({which})")
    (n_, _s, V, T, st, grid, _m), = lines
    assert -(-n // (V * T)) >= 3 * grid


# F. general-kernel configurations: (live temporaries, staged inputs, extra literal words) -> candidate
CONFIG_ROWS = [
    # k_temps, inputs, extra literals, (V, T, stages, CTAs per SM)
    (2, 1, 0, (8, 256, 1, 4)),
    (6, 1, 0, (8, 256, 1, 3)),
    (9, 1, 0, (8, 256, 2, 2)),
    (8, 4, 0, (8, 256, 1, 2)),
    (18, 1, 0, (8, 256, 2, 1)),
    (22, 4, 0, (8, 256, 1, 1)),
    (40, 1, 0, (8, 128, 2, 1)),
    (49, 4, 0, (8, 128, 1, 1)),
    (80, 1, 0, (4, 128, 2, 1)),
    (150, 1, 0, (4, 64, 2, 1)),
    (300, 1, 0, (4, 32, 2, 1)),
]
SMALL_ROWS = [(100, (4, 32, 2, 1)), (300, (4, 128, 2, 1)), (4000, (8, 256, 2, 1))]


def config_case(ek, put, n, row):
    k, inputs, lits, _want = row
    return live_temps_case(ek, put, n, k, inputs, lits)


@pytest.mark.parametrize("row", CONFIG_ROWS, ids=lambda r: "V%d_T%d_s%d_c%d" % r[3])
def test_general_kernel_configurations(clean, capfd, row):
    ek = clean
    V, T, st, c = row[3]
    n = 3 * num_sms() * c * V * T + V * T // 2 + 1          # >= 3 tiles per CTA and a ragged last tile
    put = Device(ek)
    with fast_mode(ek, False):
        cases = config_case(ek, put, n, row)
        sw = ek.debug_program()["sweeps"][0]
        assert general_config(sw, n) == row[3]
        lines, fast = run(ek, capfd, cases, f"configuration {row[3]}")
    (n_, _s, gV, gT, gst, grid, _m), = lines
    assert (gV, gT, gst, grid) == (V, T, st, num_sms() * c), lines
    assert -(-n // (V * T)) >= 3 * grid and n % (V * T) != 0


@pytest.mark.parametrize("n,want", SMALL_ROWS)
def test_small_sweep_configurations(clean, capfd, n, want):
    ek = clean
    put = Device(ek)
    with fast_mode(ek, False):
        cases = live_temps_case(ek, put, n, 4, 2)
        lines, _ = run(ek, capfd, cases, f"small sweep n={n}")
    (n_, _s, V, T, st, grid, _m), = lines
    assert (V, T, st) == want[:3] and grid == -(-n // (V * T))


# G. group splits
def test_split_many_outputs(clean, capfd):
    ek = clean
    put = Device(ek)
    cases = many_outputs_case(ek, put, (1 << 20) + 5)
    lines, _ = run(ek, capfd, cases, "300 outputs")
    assert len(lines) >= 2


@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("count", [MAX_SCALAR + 1, 2 * MAX_SCALAR + 2])
def test_split_many_scalars(clean, capfd, count, fast):
    ek = clean
    put = Device(ek)
    n = 3 * 4096 + 17
    with fast_mode(ek, fast):
        cases = scalar_case(ek, put, n, count)
        prog = ek.debug_program()
        check_scalar_plan(prog, n, count)
        lines, nfast = run(ek, capfd, cases, f"{count} scalars")
    assert len(lines) == len(prog["sweeps"])
    assert nfast == (len(lines) if fast else 0), "the scalar sweeps did not all run on the selected kernel"


def test_split_slot_pressure(clean, capfd):
    """Two results sharing 500 temporaries: together they fit no configuration, apart they do."""
    ek = clean
    put = Device(ek)
    n = 100_003
    with fast_mode(ek, False):
        cases = pressure_case(ek, put, n)
        assert len(ek.debug_program()["sweeps"]) == 2
        lines, _ = run(ek, capfd, cases, "slot pressure")
    assert len(lines) == 2


def test_split_with_side_effects(clean, capfd):
    ek = clean
    put = Device(ek)
    cases = scatter_split_case(ek, put, 65_537)
    assert scatter_halves(ek.debug_program()) >= 2, "the plain scatters into one target do not span the split"
    lines, _ = run(ek, capfd, cases, "split with scatters")
    assert len(lines) >= 2


def scatter_halves(prog):
    """Number of sweeps that hold plain scatters: at least 2 when a split separates earlier scatters into one target
    from later ones, so that the launch order decides which write wins."""
    return sum(1 for sw in prog["sweeps"] if "SCATTER_32" in ops(prog, sw))


def test_split_reduction_consumed_later(clean, capfd):
    ek = clean
    put = Device(ek)
    cases = split_reduction_case(ek, put, 1 << 18)
    phases = [s["phase"] for s in ek.debug_program()["sweeps"]]
    assert phases.count(0) >= 2 and 1 in phases
    run(ek, capfd, cases, "split with a reduction")


def test_single_root_too_large(clean, capfd):
    """One result that no configuration holds: ek_eval refuses it, launches nothing and leaves the trace as it was; after
    the caller evaluates an intermediate the same values come out exact."""
    ek = clean
    put = Device(ek)
    n = 40_009
    rng = np.random.default_rng(8)
    xn = rng.integers(-100, 100, n).astype(np.float32)
    x = put(ek.Float32, xn)
    K = 1000
    t = [x + float(i + 1) for i in range(K)]
    tn = [xn + np.float32(i + 1) for i in range(K)]
    a, an = t[0], tn[0]
    for i in range(1, K):
        a = a + t[i]; an = an + tn[i]
    b, bn = t[-1], tn[-1]
    for i in range(K - 2, -1, -1):
        b = b - t[i]; bn = bn - tn[i]
    del t
    out = a * 3.0 + b
    before = ek.stats().launches
    with pytest.raises(ek.EnokiError, match=r"insert cuda_eval\(\) to split it"):
        ek.cuda_eval()
    assert ek.stats().launches == before
    del out
    gc.collect()
    a.eval()                                   # a and b: split into two kernels, each t_i used once per kernel
    out = a * 3.0 + b
    run(ek, capfd, [("intermediate", a, an), ("result", out, an * np.float32(3) + bn)], "after the split by hand")
