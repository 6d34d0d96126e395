"""GPU: gather, scatter and scatter_add against exact host references, on every lowering the planner picks.

The planner (ek_eval.cpp: emit_var, uses_smem, mask_is_implied) lowers these operations by element width, index type,
stride, source / target size and mask: GATHER_32 / _64 / _U8 / _S8 / _U16 / _S16, GATHER_32_SMEM for tables of at most
4096 words; SCATTER_8 / 16 / 32 / 64; SCATTER_ADD_F32 / I32 / F64 / I64 as global atomics, SCATTER_ADD_F32_SMEM /
I32_SMEM (privatised bins) for targets of at most 1024 words.  Every case asserts from the plan which lowering it runs
before it evaluates, so a threshold that moves cannot silently take a case onto another path.

Buffers are guarded: each source and target is a prefix view (Type.map) of a larger device allocation whose tail holds
sentinels.  Masked-off lanes point into that tail, so a kernel that ignores the mask reads a sentinel or overwrites one
-- always inside the allocation -- and the tail is checked after every evaluation.  Index, value and mask inputs carry
a tile of padding that only a kernel without its partial-tile guard would read (in-range indices, true masks, sentinel
values: such a kernel would scatter a sentinel).

Expected values come from numpy or Python integers.  Integer sums are exact with wrap; float sums are bit-exact on
integer-valued data whose partial sums are all exactly representable (so the order of the atomics cannot matter), and
within a bound derived from the number of terms and sum |v| on random data.  Float scatter_add follows the rule of
adding every element in IEEE arithmetic in any order, which fixes the sign of zero: a -0.0 target stays -0.0 only if it
receives nothing but -0.0.

The 32-bit cases are builders (`gather_case`, `scatter_case`, `scatter_add_case`, `signed_zero_case`, `implied_case`)
taking the module and a `put(cls, array, guard)` factory; tests/test_cpu_gather_scatter.py runs them through the
planner, the assembler and the sweep-ISA emulator."""
import ctypes
import gc
import re

import numpy as np
import pytest

import test_gpu_horizontal as hz

pytestmark = pytest.mark.gpu

GUARD = 4096                     # sentinel elements past every mapped buffer (>= one sweep tile of padding)
SIZES = [1, 31, 4096, 4097, (1 << 20) + 7]
BIG = (1 << 24) + 3
TYPES = ("Bool", "UInt8", "Int8", "UInt16", "Int16", "Int32", "UInt32", "Float32", "Int64", "UInt64", "Float64")
DT = dict(hz.DTYPE, Bool=np.uint8)          # Bool as raw bytes (a borrowed mask may hold 2 or 0xff for `true`)
INDEX_TYPES = ("UInt32", "Int32", "UInt64", "Int64")
ADD_TYPES = ("Float32", "Int32", "UInt32", "Float64", "Int64", "UInt64")
BIN_COUNTS = [1, 31, 32, 33, 128, 129, 1024, 1025, 50_000]


def cls_of(ek, tname):
    return ek.Mask if tname == "Bool" else getattr(ek, tname)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8) if a.dtype == np.bool_ else a.view(hz._udt(a.dtype))


def sentinel(dt, n):
    """Guard values no correct result contains: 0x5a / 0xa5 byte patterns."""
    b = np.frombuffer(bytes([0x5a, 0xa5]) * (n * np.dtype(dt).itemsize), np.uint8)[:n * np.dtype(dt).itemsize]
    return b.copy().view(dt)


def plan_ops(ek):
    return re.findall(r"^\s+(?:init|body|fini) (\w+)", ek.debug_plan(), re.M)


class Case:
    """checks: (label, variable, expected numpy array, bound or None); plan: lowerings that must appear in the plan,
    absent: ones that must not."""
    def __init__(self):
        self.checks, self.plan, self.absent, self.keep = [], [], [], []

    def check(self, label, var, want, bound=None):
        self.checks.append((label, var, np.asarray(want), bound))

    def verify(self, got):
        bad = []
        for label, var, want, bound in self.checks:
            g = np.ascontiguousarray(got(var)).reshape(-1)[:want.size]
            if bound is not None:
                err = np.abs(g.astype(np.float64) - want.astype(np.float64))
                if not (err <= bound).all():
                    k = int(np.argmax(err - bound))
                    bad.append(f"{label}: element {k} off by {err[k]} > {bound[k] if np.ndim(bound) else bound}")
                continue
            if want.dtype.kind == "f":
                ok = (bits(g) == bits(want)) | (np.isnan(g) & np.isnan(want))
            elif label.startswith(("gather<Bool>", "scatter<Bool>")):
                ok = (g != 0) == (want != 0)        # any non-zero byte is true (a size-1 input is read as 0 / 1)
            else:
                ok = bits(g) == bits(want.astype(g.dtype) if g.dtype != want.dtype else want)
            if not ok.all():
                k = int(np.flatnonzero(~ok)[0])
                bad.append(f"{label}: {int((~ok).sum())} wrong, first at {k}: got {g[k]!r}, want {want[k]!r}")
        assert not bad, "; ".join(bad)


# ------------------------------------------------------------------ data
def index_into(rng, n, size, active, itype="UInt32"):
    """Indices of n lanes: active lanes in [0, size) with 0 and size - 1 present, masked-off lanes in the guard."""
    idx = rng.integers(0, size, n)
    if n >= 2:
        idx[0], idx[-1] = 0, size - 1
    idx = np.where(active, idx, size + rng.integers(0, GUARD, n))
    return idx.astype(DT[itype])


def masks(rng, n):
    """name -> (mask bytes or None for a literal true, which lanes are active)."""
    r = rng.random(n) < 0.6
    b = rng.choice(np.array([0, 1, 2, 0xff], np.uint8), n)
    return {"true": (None, np.ones(n, bool)), "random": (r.astype(np.uint8), r),
            "false": (np.zeros(n, np.uint8), np.zeros(n, bool)), "bytes2ff": (b, b != 0)}


def source_values(rng, tname, size):
    dt = np.dtype(DT[tname])
    if tname == "Bool":
        return rng.choice(np.array([0, 1, 2, 0xff], np.uint8), size)
    if dt.kind == "f":
        return (rng.integers(-1000, 1000, size) * 0.25).astype(dt) + dt.type(0.5)
    info = np.iinfo(dt)
    x = rng.integers(info.min, info.max, size, endpoint=True, dtype=dt)
    if dt.itemsize == 8:                 # distinct non-zero high words, top bit set on half of them
        hi = (rng.integers(1, 1 << 31, size).astype(np.uint64) | (rng.integers(0, 2, size).astype(np.uint64) << 31))
        x = ((hi << np.uint64(32)) | (x.view(np.uint64) & np.uint64(0xffffffff))).view(dt)
    if size >= 2:
        x[0], x[-1] = info.min, info.max             # -128 / -32768 sign-extend, 255 / 65535 must not
    return x


def _put_mask(ek, put, m, n):
    return ek.Mask(True) if m is None else put(ek.Mask, m, np.ones(GUARD, np.uint8))


# ------------------------------------------------------------------ builders
def gather_case(ek, put, tname, itype, n, size, seed, mask_names=("true", "random", "false", "bytes2ff")):
    """gather<tname>(source of `size`, index of type itype, mask) for each mask; narrow results also widened."""
    rng = np.random.default_rng(seed)
    T, I = cls_of(ek, tname), getattr(ek, itype)
    src = source_values(rng, tname, size)
    S = put(T, src, sentinel(src.dtype, GUARD))
    c = Case()
    c.keep.append(S)
    es = np.dtype(DT[tname]).itemsize
    smem = n > 1 and itype == "UInt32" and es == 4 and size <= 4096          # (the table is staged once per CTA)
    lowering = {1: "GATHER_U8", 2: "GATHER_U16", 4: "GATHER_32", 8: "GATHER_64"}[es]
    if tname in ("Int8", "Int16"):
        lowering = lowering.replace("_U", "_S")
    c.plan.append("GATHER_32_SMEM" if smem else lowering)
    for name, (m, active) in masks(rng, n).items():
        if name not in mask_names:
            continue
        idx = index_into(rng, n, size, active, itype)
        X = put(I, idx, np.zeros(GUARD, idx.dtype))
        r = ek.gather(T, S, X, _put_mask(ek, put, m, n))
        want = np.where(active, src[np.where(active, idx, 0).astype(np.int64)], src.dtype.type(0))
        c.check(f"gather<{tname}>[{itype}] size={size} mask={name}", r, want)
        if tname in ("Int8", "Int16"):
            c.check(f"Int32(gather<{tname}>) mask={name}", ek.Int32(r), want.astype(np.int32))
        elif tname in ("UInt8", "UInt16"):
            c.check(f"UInt32(gather<{tname}>) mask={name}", ek.UInt32(r), want.astype(np.uint32))
    return c


def scatter_case(ek, put, tname, n, seed, part, itype="UInt32"):
    """Part A: scatter of a permutation, a masked permutation and a literal value; part B: duplicate indices whose
    writers agree and a literal mask; each into its own guarded target of n elements (two evaluations keep each
    program within the fast kernel's staging budget)."""
    rng = np.random.default_rng(seed)
    T, I = cls_of(ek, tname), getattr(ek, itype)
    dt = np.dtype(DT[tname])
    c = Case()
    c.plan.append({1: "SCATTER_8", 2: "SCATTER_16", 4: "SCATTER_32", 8: "SCATTER_64"}[dt.itemsize])

    def target():
        t0 = source_values(rng, tname, n)
        return t0, put(T, t0, sentinel(dt, GUARD))

    perm = rng.permutation(n)
    v = source_values(rng, tname, n)
    V = put(T, v, sentinel(dt, GUARD))
    m = (rng.random(n) < 0.5).astype(np.uint8) * rng.choice(np.array([1, 2, 0xff], np.uint8), n)
    idx = np.where(m != 0, perm, n + rng.integers(0, GUARD, n)).astype(DT[itype])
    dup = rng.integers(0, max(1, n // 3), n)
    table = source_values(rng, tname, n)
    lit = source_values(rng, tname, 2)[1]
    if part == "A":
        P = put(I, perm.astype(DT[itype]), np.zeros(GUARD, DT[itype]))
        X, M = put(I, idx, np.zeros(GUARD, DT[itype])), put(ek.Mask, m, np.ones(GUARD, np.uint8))
        # permutation: every element written once, adjacent narrow elements by different lanes
        t0, Tg = target()
        ek.scatter(Tg, V, P)
        want = t0.copy(); want[perm] = v
        c.check(f"scatter<{tname}> permutation", Tg, want)
        # masked permutation: masked-off lanes point into the guard
        t1, Tg1 = target()
        ek.scatter(Tg1, V, X, M)
        want = t1.copy(); want[perm[m != 0]] = v[m != 0]
        c.check(f"scatter<{tname}> masked permutation", Tg1, want)
        # literal value, masked
        t3, Tg3 = target()
        ek.scatter(Tg3, T(lit.item() if tname != "Bool" else True), X, M)
        want = t3.copy(); want[perm[m != 0]] = lit if tname != "Bool" else 1
        c.check(f"scatter<{tname}> literal value", Tg3, want)
    else:
        # duplicates: lane i writes f(idx[i]), so whichever writer wins the result is the same
        t2, Tg2 = target()
        ek.scatter(Tg2, put(T, table[dup], sentinel(dt, GUARD)), put(I, dup.astype(DT[itype]), np.zeros(GUARD, DT[itype])))
        want = t2.copy(); want[dup] = table[dup]
        c.check(f"scatter<{tname}> duplicates", Tg2, want)
        # literal mask
        t4, Tg4 = target()
        ek.scatter(Tg4, V, put(I, perm[::-1].astype(DT[itype]), np.zeros(GUARD, DT[itype])), True)
        want = t4.copy(); want[perm[::-1]] = v
        c.check(f"scatter<{tname}> literal mask", Tg4, want)
    return c


def add_values(rng, tname, n, count):
    """Values whose sums are exact and exercise wrap: integer-valued floats with sum |v| well below 2^24; UInt32 values
    near 2^31 (sums pass 2^32), negative Int32 values, 64-bit values near the top of their range."""
    dt = np.dtype(DT[tname])
    if dt.kind == "f":
        return hz.integer_valued(rng, n, dt, scale=2)
    if tname == "UInt32":
        return rng.integers(1 << 31, (1 << 32) - 1, n, dtype=np.uint32)
    if tname == "Int32":
        return rng.integers(-(1 << 31), 1000, n, dtype=np.int32)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, n, endpoint=True, dtype=dt)


def add_reference(t0, idx, v, active):
    """target + every active contribution: integers with wrap, floats in the target's IEEE type (the data is such that
    the order does not matter)."""
    out = t0.copy()
    if out.dtype.kind == "f":
        with np.errstate(invalid="ignore"):          # (+inf + -inf)
            np.add.at(out, idx[active].astype(np.int64), v[active])
    else:
        u = out.view(hz._udt(out.dtype))
        np.add.at(u, idx[active].astype(np.int64), v[active].view(u.dtype))
    return out


def smem_bins(tname, count, n, itype="UInt32"):
    return n > 1 and tname in ("Float32", "Int32", "UInt32") and itype == "UInt32" and count <= 1024


def add_lowering(tname, count, n, itype="UInt32"):
    if smem_bins(tname, count, n, itype):
        return "SCATTER_ADD_F32_SMEM" if tname == "Float32" else "SCATTER_ADD_I32_SMEM"
    return {"Float32": "SCATTER_ADD_F32", "Int32": "SCATTER_ADD_I32", "UInt32": "SCATTER_ADD_I32",
            "Float64": "SCATTER_ADD_F64", "Int64": "SCATTER_ADD_I64", "UInt64": "SCATTER_ADD_I64"}[tname]


def scatter_add_case(ek, put, tname, count, n, seed, heavy=False):
    """Four scatter_adds into four non-zero targets of `count`: value array / literal x mask array / literal; with
    `heavy`, every lane of the first two hits one bin."""
    rng = np.random.default_rng(seed)
    T, I = getattr(ek, tname), ek.UInt32
    dt = np.dtype(DT[tname])
    c = Case()
    c.plan.append(add_lowering(tname, count, n))
    lit = dt.type(3) if dt.kind == "f" else hz._wrap(-7, dt)          # (unsigned: 2^w - 7, the sums wrap)
    for k, (vkind, mkind) in enumerate([("array", "array"), ("literal", "array"), ("array", "literal"), ("literal", "literal")]):
        t0 = (hz.integer_valued(rng, count, dt, scale=64) if dt.kind == "f" else add_values(rng, tname, count, count))
        if count >= 2 and dt.kind == "f":
            t0[0] = dt.type(5.0)
        Tg = put(T, t0, sentinel(dt, GUARD))
        active = np.ones(n, bool) if mkind == "literal" else rng.random(n) < 0.7
        idx = np.full(n, count // 2) if heavy and k < 2 else rng.integers(0, count, n)
        idx = np.where(active, idx, count + rng.integers(0, GUARD, n)).astype(np.uint32)
        if vkind == "array":
            v = add_values(rng, tname, n, count)
            V = put(T, v, sentinel(dt, GUARD))
        else:
            if dt.kind == "f" and n * 3 >= 1 << 23:
                continue                      # (a literal 3.0 on every lane would pass the exactness bound)
            v = np.full(n, lit, dt)
            V = T(lit.item())
        M = True if mkind == "literal" else put(ek.Mask, active.astype(np.uint8) * rng.choice(np.array([1, 2, 0xff], np.uint8), n),
                                                np.ones(GUARD, np.uint8))
        ek.scatter_add(Tg, V, put(I, idx, np.zeros(GUARD, np.uint32)), M)
        c.check(f"scatter_add<{tname}> count={count} value={vkind} mask={mkind}{' heavy' if heavy and k < 2 else ''}",
                Tg, add_reference(t0, idx, v, active))
    return c


def signed_zero_case(ek, put, count, n, seed):
    """Float32 scatter_add: -0.0 targets with +0.0 contributions and with contributions that cancel, -0.0 into +0.0 and
    into -0.0, bins that receive nothing, +-inf and NaN (+inf and -inf into one bin gives NaN).  Padding lanes are
    masked off and point into the guard."""
    assert count >= 12
    rng = np.random.default_rng(seed)
    nz, pz = np.float32(-0.0), np.float32(0.0)
    t0 = np.full(count, 7.0, np.float32)
    t0[:12] = [nz, nz, pz, nz, nz, pz, 1.0, 1.0, 2.0, -1.0, nz, pz]
    contrib = [(0, pz), (0, pz), (1, 4.0), (1, -4.0), (1, 2.0), (1, -2.0), (2, nz), (2, nz), (3, nz), (3, nz),
               (6, np.inf), (7, np.inf), (7, -np.inf), (8, np.nan), (8, 1.0), (9, -np.inf), (9, 3.0)]
    # bins 4, 5, 10, 11 receive nothing; the rest of the target gets +1 / -1 pairs and single +1 / -1
    rest = rng.integers(12, count, min(3 * count, n - len(contrib) - 100))
    contrib += [(int(b), np.float32(s)) for b, s in zip(rest, rng.choice(np.array([1.0, -1.0], np.float32), rest.size))]
    contrib = [contrib[k] for k in rng.permutation(len(contrib))]
    m = len(contrib)
    idx = np.array([b for b, _ in contrib[:m]] + list(count + rng.integers(0, GUARD, n - m)), np.uint32)
    v = np.array([x for _, x in contrib[:m]] + [np.float32(123.0)] * (n - m), np.float32)
    active = np.arange(n) < m
    c = Case()
    c.plan.append(add_lowering("Float32", count, n))
    Tg = put(ek.Float32, t0, sentinel(np.float32, GUARD))
    ek.scatter_add(Tg, put(ek.Float32, v, sentinel(np.float32, GUARD)), put(ek.UInt32, idx, np.zeros(GUARD, np.uint32)),
                   put(ek.Mask, active.astype(np.uint8), np.ones(GUARD, np.uint8)))
    want = add_reference(t0, idx, v, active)
    assert np.signbit(want[4]) and not np.signbit(want[0]) and not np.signbit(want[1]) and np.isnan(want[7])
    c.check(f"signed zeros count={count} n={n}", Tg, want)
    return c, m


def implied_case(ek, put, kind, n, seed, count=31):
    """Gather and scatter_add with a mask `idx < L`: kind 'equal' (L = count), 'above' (count + 5), 'below' (count - 3),
    'shared' (L = count, the comparison also selects a second output) or 'signed' (an Int32 index)."""
    rng = np.random.default_rng(seed)
    signed = kind == "signed"
    I = ek.Int32 if signed else ek.UInt32
    L = {"equal": count, "above": count + 5, "below": count - 3, "shared": count, "signed": count}[kind]
    idx = rng.integers(0, count + 40, n)
    if kind == "above":                  # (lanes the mask lets through must stay inside the target)
        idx = np.where((idx >= count) & (idx < L), idx - count, idx)
    idx = idx.astype(np.int32 if signed else np.uint32)
    tab = (np.arange(count, dtype=np.float32) * 0.5 + 1.0)
    c = Case()
    S = put(ek.Float32, tab, sentinel(np.float32, GUARD))
    bins0 = rng.integers(0, 100, count).astype(np.uint32)
    B = put(ek.UInt32, bins0, sentinel(np.uint32, GUARD))
    c.keep.append(S)
    X = put(I, idx, np.zeros(GUARD, idx.dtype))
    M = X < I(L)
    r = ek.gather(ek.Float32, S, X, M)
    ek.scatter_add(B, ek.UInt32(1), X, M)
    active = idx.astype(np.int64) < L
    inr = active & (idx.astype(np.int64) < count)
    c.check(f"implied {kind}: gather", r, np.where(inr, tab[np.where(inr, idx, 0).astype(np.int64)], np.float32(0)))
    want = bins0.copy(); np.add.at(want, idx[active].astype(np.int64), np.uint32(1))
    c.check(f"implied {kind}: bins", B, want)
    if kind == "shared":
        s = ek.select(M, ek.UInt32(1), ek.UInt32(2))
        c.check("implied shared: select", s, np.where(active, 1, 2).astype(np.uint32))
    if signed:
        c.plan += ["GATHER_32", "SCATTER_ADD_I32", "LT_I32"]
        c.absent += ["GATHER_32_SMEM", "SCATTER_ADD_I32_SMEM"]
    else:
        c.plan += ["GATHER_32_SMEM", "SCATTER_ADD_I32_SMEM"]
        (c.absent if kind in ("equal", "above") else c.plan).append("LT_U32")
    return c


# ------------------------------------------------------------------ device staging and the runner
class Guarded:
    """put(cls, array, guard): a Type.map view of the array in a device allocation followed by `guard`."""
    def __init__(self, ek):
        self.ek, self.bufs = ek, []

    def __call__(self, cls, arr, guard):
        lib = self.ek.lib()
        arr = np.ascontiguousarray(arr)
        host = np.concatenate([arr, np.asarray(guard).astype(arr.dtype)])
        p = lib.ek_malloc(host.nbytes)
        lib.ek_memcpy_to_device(p, host.ctypes.data, host.nbytes)
        self.bufs.append((p, host, arr.nbytes))
        return cls.map(p, len(arr))

    def check_guards(self):
        lib = self.ek.lib()
        lib.ek_sync()
        for p, host, nb in self.bufs:
            tail = np.empty(host.nbytes - nb, np.uint8)
            lib.ek_memcpy_from_device(tail.ctypes.data, p + nb, tail.nbytes)
            bad = np.flatnonzero(tail != host.view(np.uint8)[nb:])
            assert bad.size == 0, f"guard overwritten {bad.size} bytes, first {bad[0]} bytes past the end"

    def free(self):
        """Drop the scatters a failed case left pending, evaluate whatever recorded work is still alive (a failed
        case's gathers, kept by its traceback) while the buffers it reads exist, and only then free them: nothing
        recorded over these buffers can run after they are gone."""
        lib = self.ek.lib()
        gc.collect()
        lib.ek_debug_discard_side_effects()
        try:
            self.ek.cuda_eval()
        except self.ek.EnokiError:
            pass
        lib.ek_sync()
        for p, _, _ in self.bufs:
            lib.ek_free(p)
        self.bufs = []


def got_gpu(var):
    a = var.numpy()
    return a.view(np.uint8) if a.dtype == np.bool_ else a


def check_plan(ek, case):
    ops = plan_ops(ek)
    for op in case.plan:
        assert op in ops, f"{op} not in the plan {sorted(set(ops))}"
    for op in case.absent:
        assert op not in ops, f"{op} in the plan {sorted(set(ops))}"
    return ops


def run(ek, build, mode, expect_fast):
    """Record the case, check its plan, evaluate it in one cuda_eval(), check the results, the guards and which kernel
    ran."""
    st, case = Guarded(ek), None
    try:
        with hz.kernel(ek, mode):
            case = build(st)
            check_plan(ek, case)
            ek.lib().ek_stats_reset()
            ek.cuda_eval()
            fast = ek.stats().fast_launches
            case.verify(got_gpu)
            st.check_guards()
        if mode == "general":
            assert fast == 0, "the fast kernel ran although it was disabled"
        elif expect_fast:
            assert fast >= 1, "the fast kernel did not run"
    finally:
        case = None                      # (a traceback keeps this frame: it must not keep the case's variables)
        st.free()


def fast_expected(tname, itype, n):
    return tname in ("Float32", "Int32", "UInt32") and itype in ("UInt32", "Int32") and n > 4096


def modes(tname, itype="UInt32"):
    return ("fast", "general") if tname in ("Float32", "Int32", "UInt32") and itype in ("UInt32", "Int32") else ("default",)


# ------------------------------------------------------------------ gather
GATHER_PARAMS = [(t, i, m) for t in TYPES for i in INDEX_TYPES for m in modes(t, i)]


@pytest.mark.parametrize("n", [31, 4097])
@pytest.mark.parametrize("tname,itype,mode", GATHER_PARAMS)
def test_gather(gpu, tname, itype, mode, n):
    for size in (1, 31, 4096, 4097, 100_003):
        run(gpu, lambda put: gather_case(gpu, put, tname, itype, n, size, seed=n + size), mode,
            mode == "fast" and fast_expected(tname, itype, n))


@pytest.mark.parametrize("n", [1, 4096, (1 << 20) + 7])
@pytest.mark.parametrize("tname,itype,mode", [("Float32", "UInt32", "fast"), ("Float32", "UInt32", "general"),
                                              ("Int32", "Int32", "fast"), ("Int8", "UInt32", "default"),
                                              ("UInt16", "Int64", "default"), ("UInt64", "UInt32", "default")])
def test_gather_sizes(gpu, tname, itype, mode, n):
    for size in (31, 4096, 4097):
        run(gpu, lambda put: gather_case(gpu, put, tname, itype, n, size, seed=n ^ size), mode,
            mode == "fast" and fast_expected(tname, itype, n))


@pytest.mark.parametrize("tname,size", [("Float32", 4096), ("Float32", 4097), ("Int64", 5000), ("UInt8", 300),
                                        ("Int8", 300), ("UInt16", 70_000), ("Int16", 70_000)])
def test_gather_2_24_plus_3(gpu, tname, size):
    """One 2^24 + 3 case per lowering: GATHER_32_SMEM, GATHER_32, GATHER_64, GATHER_U8 / S8 / U16 / S16."""
    mode = "fast" if tname == "Float32" else "default"
    run(gpu, lambda put: gather_case(gpu, put, tname, "UInt32", BIG, size, seed=size, mask_names=("random",)), mode,
        mode == "fast")


# ------------------------------------------------------------------ scatter
SCATTER_TYPES = ("Bool", "UInt8", "Int16", "UInt16", "Float32", "Int32", "UInt32", "Int64", "Float64", "UInt64")


# (a plain scatter is recorded with type UInt64, as in the reference, which marks its program 64-bit: it runs on the
# general kernel with high planes whatever it moves)
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("tname", SCATTER_TYPES)
def test_scatter(gpu, tname, n):
    for part in "AB":
        run(gpu, lambda put: scatter_case(gpu, put, tname, n, seed=n, part=part), "default", False)


@pytest.mark.parametrize("tname", ["UInt8", "Int16", "Float32", "Float64"])
def test_scatter_2_24_plus_3(gpu, tname):
    for part in "AB":
        run(gpu, lambda put: scatter_case(gpu, put, tname, BIG, seed=5, part=part), "default", False)


@pytest.mark.parametrize("itype", ["Int32", "UInt64", "Int64"])
@pytest.mark.parametrize("tname", ["UInt8", "Float32", "UInt64"])
def test_scatter_index_types(gpu, tname, itype):
    for part in "AB":
        run(gpu, lambda put: scatter_case(gpu, put, tname, 4097, seed=9, part=part, itype=itype), "default", False)


# ------------------------------------------------------------------ scatter_add
@pytest.mark.parametrize("n", [31, 4097])
@pytest.mark.parametrize("count", BIN_COUNTS)
@pytest.mark.parametrize("tname,mode", [(t, m) for t in ADD_TYPES for m in modes(t)])
def test_scatter_add(gpu, tname, mode, count, n):
    run(gpu, lambda put: scatter_add_case(gpu, put, tname, count, n, seed=count + n), mode,
        mode == "fast" and fast_expected(tname, "UInt32", n))
    run(gpu, lambda put: scatter_add_case(gpu, put, tname, count, n, seed=count * n, heavy=True), mode,
        mode == "fast" and fast_expected(tname, "UInt32", n))


@pytest.mark.parametrize("count", [1, 32, 33, 129, 1025, 50_000])
@pytest.mark.parametrize("tname,mode", [(t, m) for t in ADD_TYPES for m in modes(t)])
def test_scatter_add_large(gpu, tname, mode, count):
    n = (1 << 20) + 7
    run(gpu, lambda put: scatter_add_case(gpu, put, tname, count, n, seed=count, heavy=count in (1, 129)), mode,
        mode == "fast" and fast_expected(tname, "UInt32", n))


@pytest.mark.parametrize("tname,count", [("Float32", 31), ("Int32", 129), ("Float32", 50_000), ("UInt32", 1025),
                                         ("Float64", 129), ("Int64", 1000)])
def test_scatter_add_2_24_plus_3(gpu, tname, count):
    """One 2^24 + 3 case per lowering: F32_SMEM, I32_SMEM, F32, I32, F64, I64."""
    mode = "fast" if tname in ("Float32", "Int32", "UInt32") else "default"
    run(gpu, lambda put: scatter_add_case(gpu, put, tname, count, BIG, seed=count), mode, mode == "fast")


@pytest.mark.parametrize("mode", ["fast", "general"])
@pytest.mark.parametrize("count", [31, 129, 1025, 50_000])
@pytest.mark.parametrize("tname", ["Float32", "Float64"])
def test_scatter_add_rounding_bound(gpu, tname, count, mode):
    """Random non-integer values: each bin's result is a summation tree over its target and its k contributions (the
    extra -0.0 / +0.0 leaves of the privatised copies are exact), so its error is at most 1.01 * k * eps * (|t| + sum
    |v|).  With thousands of terms per bin that bound is far wider than one contribution, so this only guards against
    gross errors of the float paths on general data; lost or duplicated contributions are caught by the exact
    integer-valued cases."""
    if tname == "Float64" and mode == "fast":
        pytest.skip("64-bit programs run on the general kernel only")
    ek = gpu
    n = (1 << 20) + 7
    dt = DT[tname]
    rng = np.random.default_rng(count)
    t0 = rng.uniform(-10, 10, count).astype(dt)
    v = (rng.uniform(-1, 1, n) * 3.7).astype(dt)
    idx = rng.integers(0, count, n).astype(np.uint32)
    exact = t0.astype(np.float64).copy(); np.add.at(exact, idx, v.astype(np.float64))
    mag = np.abs(t0.astype(np.float64)); np.add.at(mag, idx, np.abs(v.astype(np.float64)))
    k = np.bincount(idx, minlength=count)
    eps = 2.0 ** -24 if dt == np.float32 else 2.0 ** -53
    bound = 1.01 * np.maximum(k, 1) * eps * mag

    def build(put):
        c = Case()
        c.plan.append(add_lowering(tname, count, n))
        Tg = put(getattr(ek, tname), t0, sentinel(dt, GUARD))
        ek.scatter_add(Tg, put(getattr(ek, tname), v, sentinel(dt, GUARD)), put(ek.UInt32, idx, np.zeros(GUARD, np.uint32)))
        c.check(f"scatter_add<{tname}> random count={count}", Tg, exact, bound)
        return c
    run(ek, build, "default" if tname == "Float64" else mode, mode == "fast" and tname == "Float32")


@pytest.mark.parametrize("mode", ["fast", "general"])
@pytest.mark.parametrize("n", [4097, 100_003])
@pytest.mark.parametrize("count", [31, 32, 33, 129, 1024, 1025, 50_000])
def test_scatter_add_signed_zero(gpu, count, n, mode):
    """Float bins start at -0.0 and skip only bins still holding -0.0 bits: per-thread copies (<= 32 bins), shared
    atomics (33..1024) and the global atomics agree with the IEEE sum of every element."""
    run(gpu, lambda put: signed_zero_case(gpu, put, count, n, seed=count)[0], mode, mode == "fast")


# ------------------------------------------------------------------ the implied mask
@pytest.mark.parametrize("mode", ["fast", "general"])
@pytest.mark.parametrize("n", [4097, 100_003])
@pytest.mark.parametrize("kind", ["equal", "above", "below", "shared", "signed"])
def test_implied_mask(gpu, kind, n, mode):
    run(gpu, lambda put: implied_case(gpu, put, kind, n, seed=n), mode, mode == "fast")


# ------------------------------------------------------------------ strides (ek_trace_append directly)
def _strided(ek, st, op, tname, stride, nrec, n, seed):
    """gather / scatter of a field of type tname at byte offset `stride // 2` rounded to the element size, from / into
    nrec interleaved records of `stride` bytes."""
    lib = ek.lib()
    rng = np.random.default_rng(seed)
    dt = np.dtype(DT[tname])
    es = dt.itemsize
    off = (stride // 2) // es * es
    raw = rng.integers(0, 256, nrec * stride, dtype=np.uint8)
    rec = st(ek.UInt8, raw, np.zeros(GUARD, np.uint8))
    base = ek.lib().ek_var_ptr(rec.index) + off
    field = lambda r: np.ndarray((nrec,), dt, r.data, off, (stride,))
    idx = rng.integers(0, nrec, n).astype(np.uint32)
    m = rng.random(n) < 0.7
    X = st(ek.UInt32, np.where(m, idx, 0).astype(np.uint32), np.zeros(GUARD, np.uint32))
    M = st(ek.Mask, m.astype(np.uint8), np.ones(GUARD, np.uint8))
    T = getattr(ek, tname)
    assert lib.ek_set_scatter_gather_operand(rec.index, op == "GATHER") == 0
    ptr = lib.ek_var_register_ptr(base)
    try:
        if op == "GATHER":
            h = lib.ek_trace_append(T.Type, ek.OP["GATHER"], ptr, X.index, M.index, stride)
            assert h, lib.ek_last_error()
            r = T.from_index(h)
            want = np.where(m, field(raw)[idx], dt.type(0))
            return rec, r, want
        perm = rng.permutation(nrec)[:n] if n <= nrec else None
        X2 = st(ek.UInt32, perm.astype(np.uint32), np.zeros(GUARD, np.uint32))
        v = rng.integers(0, 1 << 62, n).astype(np.uint64).view(np.uint8)[:n * es].view(dt)
        V = st(T, v, np.zeros(GUARD, dt))
        h = lib.ek_trace_append(ek.EK_UINT64, ek.OP["SCATTER"], ptr, X2.index, M.index, (stride << 32) | V.index)
        assert h, lib.ek_last_error()
        lib.ek_var_mark_side_effect(h)
        lib.ek_var_mark_dirty(rec.index)
        want = raw.copy()
        field(want)[perm[m]] = v[m]
        return rec, rec, want
    finally:
        lib.ek_dec_ref_ext(ptr)
        lib.ek_set_scatter_gather_operand(0, 0)


@pytest.mark.parametrize("op", ["GATHER", "SCATTER"])
@pytest.mark.parametrize("tname,stride", [("UInt32", 8), ("Float32", 12), ("Int32", 16), ("UInt64", 16),
                                          ("Float64", 24), ("UInt32", 32764)])
def test_strides(gpu, op, tname, stride):
    ek = gpu
    nrec = 300 if stride > 1000 else 5000
    n = 257 if op == "SCATTER" else 4097
    st = Guarded(ek)
    try:
        rec, out, want = _strided(ek, st, op, tname, stride, nrec, n, seed=stride)
        ek.cuda_eval()
        got = out.numpy()
        assert (bits(got) == bits(want)).all(), int(np.flatnonzero(bits(got) != bits(want))[0])
        st.check_guards()
        del rec, out
    finally:
        st.free()


def stride_rejection(ek, base):
    """Strides that do not fit the 15-bit field are refused with an error naming the limit; 32764 is accepted.  `base`
    addresses at least 16 * 32768 bytes (enough for any stride that wraps).  Nothing recorded here is evaluated: a
    refused append returns no handle, and whatever an append does return is released at once (it is no side effect,
    so it leaves the trace with its last reference)."""
    lib = ek.lib()
    X, M = ek.UInt32.arange(16), ek.Mask(True)
    ptr = lib.ek_var_register_ptr(base)

    def append(t, op, imm):
        h = lib.ek_trace_append(t, ek.OP[op], ptr, X.index, M.index, imm)
        if h:
            lib.ek_dec_ref_ext(h)
        return h
    try:
        for stride in (32768, 40000, 1 << 20):
            assert not append(ek.EK_UINT32, "GATHER", stride), f"gather stride {stride} accepted"
            assert b"32767" in lib.ek_last_error()
            for op, t in (("SCATTER", ek.EK_UINT64), ("SCATTER_ADD", ek.EK_UINT32)):
                assert not append(t, op, (stride << 32) | X.index), f"{op} stride {stride} accepted"
                assert b"32767" in lib.ek_last_error()
        assert append(ek.EK_UINT32, "GATHER", 32764), lib.ek_last_error()
    finally:
        lib.ek_dec_ref_ext(ptr)
        del X, M
        gc.collect()
        lib.ek_debug_discard_side_effects()
        assert ek.debug_plan() == "", "a recorded gather or scatter is still pending"


def test_stride_rejection(gpu):
    lib = gpu.lib()
    p = lib.ek_malloc(16 * 32768)
    try:
        stride_rejection(gpu, p)
    finally:
        lib.ek_sync()
        lib.ek_free(p)


# ------------------------------------------------------------------ order within one evaluation
@pytest.mark.parametrize("mode", ["fast", "general"])
@pytest.mark.parametrize("n", [4097, 100_003])
def test_order(gpu, n, mode):
    ek = gpu
    rng = np.random.default_rng(n)
    st = Guarded(ek)
    try:
        with hz.kernel(ek, mode):
            # a gather from a target that was scattered into sees the update
            t0 = np.arange(n, dtype=np.float32)
            Tg = st(ek.Float32, t0, sentinel(np.float32, GUARD))
            perm = rng.permutation(n).astype(np.uint32)
            P = st(ek.UInt32, perm, np.zeros(GUARD, np.uint32))
            ek.scatter(Tg, ek.Float32(-1.0), P, st(ek.Mask, (perm % 3 == 0).astype(np.uint8), np.ones(GUARD, np.uint8)))
            g = ek.gather(ek.Float32, Tg, ek.UInt32.arange(n))
            want = t0.copy(); want[perm[perm % 3 == 0]] = -1.0
            assert (g.numpy() == want).all()
            # two scatter_adds into one small target and a table gather + bin scatter_add, all in one sweep
            cnt = 31
            b0 = rng.integers(0, 100, cnt).astype(np.uint32)
            B = st(ek.UInt32, b0, sentinel(np.uint32, GUARD))
            tab = rng.integers(-50, 50, cnt).astype(np.float32)
            S = st(ek.Float32, tab, sentinel(np.float32, GUARD))
            H = st(ek.Float32, np.zeros(cnt, np.float32), sentinel(np.float32, GUARD))
            i1 = rng.integers(0, cnt, n).astype(np.uint32); i2 = rng.integers(0, cnt, n).astype(np.uint32)
            I1, I2 = st(ek.UInt32, i1, np.zeros(GUARD, np.uint32)), st(ek.UInt32, i2, np.zeros(GUARD, np.uint32))
            ek.scatter_add(B, ek.UInt32(1), I1)
            ek.scatter_add(B, ek.UInt32(1000), I2)
            w = ek.gather(ek.Float32, S, I1)
            ek.scatter_add(H, w, I2)
            prog = ek.debug_program()
            wide = [s for s in prog["sweeps"] if s["n"] == n]
            assert len(wide) == 1
            ops = plan_ops(ek)
            assert ops.count("SCATTER_ADD_I32_SMEM") == 2 and "GATHER_32_SMEM" in ops and "SCATTER_ADD_F32_SMEM" in ops
            ek.cuda_eval()
            wb = b0.copy(); np.add.at(wb, i1, 1); np.add.at(wb, i2, 1000)
            wh = np.zeros(cnt, np.float64); np.add.at(wh, i2, tab[i1].astype(np.float64))
            assert (B.numpy() == wb).all()
            assert (w.numpy() == tab[i1]).all()
            assert (H.numpy() == wh.astype(np.float32)).all()
            st.check_guards()
            del g, w
    finally:
        st.free()


# ------------------------------------------------------------------ tape edges (raw C ABI)
def _tape(ek, tname):
    return ek.lib(), getattr(ek, tname), getattr(ek, "EK_" + tname.upper()), DT[tname]


def _grad(ek, L, T, et, leaf, node, g):
    G = T.copy(g)
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


@pytest.mark.parametrize("permute", [0, 1])
@pytest.mark.parametrize("size", [31, 1024, 1025, 5000])
@pytest.mark.parametrize("tname", ["Float32", "Float64"])
def test_tape_gather_gradient(gpu, tname, size, permute):
    """The adjoint of a gather is a scatter_add of the node's gradient into the source's (a plain scatter with
    `permute`), masked lanes excluded; F32 sources of <= 1024 entries take the shared-memory bins."""
    ek = gpu
    L, T, et, dt = _tape(ek, tname)
    n = 4097
    rng = np.random.default_rng(size + permute)
    if permute:                          # each source element is gathered by at most one lane
        off = rng.permutation(size)[:n]
        n = off.size
    else:
        off = rng.integers(0, size, n)
    off = off.astype(np.uint32)
    m = rng.random(n) < 0.7
    g = rng.integers(-20, 20, n).astype(dt)
    leaf = L.ek_tape_append_leaf(et, size)
    src = ctypes.c_uint32(leaf)
    assert L.ek_tape_set_scatter_gather_operand(et, ctypes.byref(src), size, permute) == 0
    O, M = ek.UInt32.copy(off), ek.Mask.copy(m)
    node = L.ek_tape_append_gather(et, O.index, M.index)
    assert L.ek_tape_set_scatter_gather_operand(et, None, 0, 0) == 0
    assert node, L.ek_last_error()
    del O, M
    got = _grad(ek, L, T, et, leaf, node, g)
    want = np.zeros(size, dt)
    if permute:
        want[off[m]] = g[m]
    else:
        np.add.at(want, off[m].astype(np.int64), g[m])
    assert (bits(got) == bits(want)).all(), int(np.flatnonzero(bits(got) != bits(want))[0])


@pytest.mark.parametrize("source", ["array", "size1"])
@pytest.mark.parametrize("scatter_add", [0, 1])
@pytest.mark.parametrize("tname", ["Float32", "Float64"])
def test_tape_scatter_gradient(gpu, tname, scatter_add, source):
    """The adjoint of a scatter / scatter_add is a masked gather of the target's gradient; from a size-1 source the
    gathered values are summed (hsum)."""
    ek = gpu
    L, T, et, dt = _tape(ek, tname)
    size, n = 1025, 4097
    rng = np.random.default_rng(scatter_add)
    off = (rng.integers(0, size, n) if scatter_add else rng.permutation(n) % size).astype(np.uint32)
    m = rng.random(n) < 0.6
    gt = rng.integers(-20, 20, size).astype(dt)
    leaf = L.ek_tape_append_leaf(et, 1 if source == "size1" else n)
    tgt = ctypes.c_uint32(0)
    assert L.ek_tape_set_scatter_gather_operand(et, ctypes.byref(tgt), size, 0) == 0
    O, M = ek.UInt32.copy(off), ek.Mask.copy(m)
    assert L.ek_tape_append_scatter(et, leaf, O.index, M.index, scatter_add) == 0, L.ek_last_error()
    assert L.ek_tape_set_scatter_gather_operand(et, None, 0, 0) == 0
    node = tgt.value
    assert node
    del O, M
    got = _grad(ek, L, T, et, leaf, node, gt)
    per_lane = np.where(m, gt[off], dt(0))
    want = np.array([per_lane.astype(np.float64).sum()], dt) if source == "size1" else per_lane
    assert (bits(got) == bits(want)).all(), (got[:4], want[:4])
