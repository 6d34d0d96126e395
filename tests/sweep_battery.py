"""The programs that pin the two sweep kernels to each other: the general kernel (ek_sweep.cu, every type) and the fast
kernel for 32-bit programs (ek_sweep_fast.cu).  Both run the same device functions for every operation (ek_math.cuh),
so evaluated with ek_set_fast_mode(0) and then with ek_set_fast_mode(1), every element-wise and integer result must
agree bit for bit; float reductions and float scatter_add totals are folded in a different order by the two kernels
and agree within a tolerance.

battery(upload, evaluate) records every program through the Python mirror (or ek_trace_append where the mirror has no
direct form) and returns one Record per kept value:
  upload(cls, ndarray)  -> an array of type cls holding the data (on the GPU: cls.copy; on the host: a fake mapping)
  evaluate(var=None)    -> evaluates everything pending and returns var's values as an ndarray (None on the host)
Record.kind 0 compares bytes; kind 1 compares f32 values with |a - b| <= tol * scale, where a scale of 0 stands for the
largest finite |a| of the array.

Inputs come from a 64-bit xorshift generator, so the programs and their data are a fixed function of the seeds.
Where one expression records several nodes, they are recorded last operand first: the planned programs depend on the
recording order, so it is part of the battery.
"""
import collections

import numpy as np

import enoki_b200 as ek
from enoki_b200 import Float32, Int32, Mask, UInt32

Record = collections.namedtuple("Record", "name array kind tol scale")

_M64 = (1 << 64) - 1


def _xorshift(s):
    s ^= (s << 13) & _M64
    s ^= s >> 7
    s ^= (s << 17) & _M64
    return s


def _apply(cols, s):
    """The GF(2) matrix with columns `cols` times the 64-bit vector s."""
    r = 0
    for c in cols:
        if not s:
            break
        if s & 1:
            r ^= c
        s >>= 1
    return r


# xorshift is linear over GF(2): _JUMP[j] advances a state by 2^j steps
_JUMP = [[_xorshift(1 << i) for i in range(64)]]
for _ in range(31):
    _JUMP.append([_apply(_JUMP[-1], c) for c in _JUMP[-1]])


def _jump(s, k):
    j = 0
    while k:
        if k & 1:
            s = _apply(_JUMP[j], s)
        k >>= 1
        j += 1
    return s


def _uniform(lo, hi, x):
    """lo + (hi - lo) * (the low 24 bits of x) / 2^24, every step rounded to float32."""
    f = np.asarray(np.asarray(x) & 0xFFFFFF).astype(np.float32)
    return np.float32(lo) + np.float32(hi - lo) * f / np.float32(16777216)


class Rng:
    def __init__(self, seed):
        self.s = (seed * 0x9E3779B97F4A7C15 + 0x1234567) & _M64

    def next(self):
        self.s = _xorshift(self.s)
        return (self.s >> 16) & 0xFFFFFFFF

    def below(self, n):
        return self.next() % n

    def uniform(self, lo, hi):
        return _uniform(lo, hi, self.next())

    def take(self, m):
        """The next m values of next() as uint32, generated on interleaved lanes of 2^k consecutive steps each."""
        steps = 1 << max(0, (m - 1).bit_length() + 1) // 2
        lanes = -(-m // steps)
        starts = [self.s]
        for _ in range(lanes - 1):
            starts.append(_jump(starts[-1], steps))
        s = np.array(starts, np.uint64)
        out = np.empty((lanes, steps), np.uint32)
        for t in range(steps):
            s ^= s << np.uint64(13)
            s ^= s >> np.uint64(7)
            s ^= s << np.uint64(17)
            out[:, t] = s >> np.uint64(16)
        self.s = _jump(self.s, m)
        return out.reshape(-1)[:m]

    def uniforms(self, lo, hi, m):
        return _uniform(lo, hi, self.take(m))


def _op(cls, op, *args):
    """One node through the C ABI: reductions are recorded even over a size-1 operand, which the mirror returns as is."""
    h = ek.lib().ek_trace_append(cls.Type, ek.OP[op], *[a.index for a in args], *[0] * (3 - len(args)), 0)
    if not h:
        raise ek.EnokiError(ek.lib().ek_last_error().decode())
    return cls.from_index(h)


def _magnitude(a):
    """Sum of the finite |a| (the scale of a float sum); 0 when there are no values (on the host)."""
    return 0.0 if a is None else float(np.abs(a[np.isfinite(a)].astype(np.float64)).sum())


class _Battery:
    def __init__(self, upload, evaluate):
        self.upload, self.evaluate, self.records = upload, evaluate, []

    def keep(self, name, var, kind=0, tol=1e-5, scale=0.0):
        self.records.append(Record(name, self.evaluate(var), kind, tol, scale))
        return self.records[-1]

    # ------------------------------------------------------------------ random expression DAGs
    def random_dag(self, seed, n):
        """A random DAG over f32 / u32 values (the shape of test_gpu_fuzz.py), a few outputs kept, reductions on top."""
        rng = Rng(seed)
        hf = rng.uniforms(-4, 4, 3 * n).reshape(3, n)
        pairs = rng.take(4 * n).reshape(2, n, 2)
        hu = pairs[..., 0] ^ (pairs[..., 1] << np.uint32(16))
        hf[0][0] = 0.0; hf[0][1 % n] = -0.0; hf[1][2 % n] = np.inf; hf[2][3 % n] = np.nan; hf[1][4 % n] = np.float32(1e-41)
        sc = rng.uniform(-2, 2)
        su = 1 + rng.below(99)
        fl = [self.upload(Float32, a) for a in hf] + [self.upload(Float32, np.array([sc], np.float32))]
        it = [self.upload(UInt32, a) for a in hu] + [self.upload(UInt32, np.array([su], np.uint32))]
        for _ in range(8 + rng.below(32)):
            _dag_node(rng, fl, it)
        keep_f = [fl[rng.below(len(fl))] for _ in range(4)]
        keep_i = [it[rng.below(len(it))] for _ in range(3)]
        del fl, it
        red_i = _op(UInt32, "HSUM", keep_i[0])
        red_f = _op(Float32, "HSUM", keep_f[0])
        # (x86 max with a NaN operand returns the second operand, so a maximum over data with NaNs depends on the fold
        # order, which differs between the kernels: take it over the NaN-free values)
        zero = Float32(0.0)
        red_m = _op(Float32, "HMAX", ek.select(keep_f[1].eq_(keep_f[1]), keep_f[1], zero))
        del zero
        self.evaluate()
        kept_f = [self.keep(f"dag{seed}.f{k}", v) for k, v in enumerate(keep_f)]
        for k, v in enumerate(keep_i):
            self.keep(f"dag{seed}.i{k}", v)
        if keep_i[0].size() > 1:
            self.keep(f"dag{seed}.hsum_u32", red_i)
        if keep_f[0].size() > 1:       # the kernels fold in different orders: relative to the sum of magnitudes
            self.keep(f"dag{seed}.hsum_f32", red_f, 1, 4e-6, _magnitude(kept_f[0].array) + 1e-30)
        if keep_f[1].size() > 1:
            self.keep(f"dag{seed}.hmax_f32", red_m)

    # ------------------------------------------------------------------ directed programs
    def directed(self, n):
        rng = Rng(4242 + n)
        h = rng.uniforms(-4, 4, 4 * n).reshape(n, 4).T
        x = [self.upload(Float32, np.ascontiguousarray(a)) for a in h]
        self.c2(x)
        for bound in (30, 31):
            self.c3(x, bound)
        self.global_gather_scatter(rng, n, x)
        self.masks(x)
        self.integers(n, x)
        self.reductions(x)

    def c2(self, x):
        """C2 (bench.py): fused arith + exp / sin / sqrt chain, with the fused hsum."""
        x0, x1, x2, x3 = x
        t = ek.fmadd(x0, x1, x2)
        u = ek.exp(-(t * t))
        v = ek.sin(ek.fmadd(x3, u, x0))
        out = ek.fmadd(v, x1, ek.sqrt(abs(t)))
        s = _op(Float32, "HSUM", out)
        del t, u, v
        r = self.keep("c2.out", out)
        self.keep("c2.hsum", s, 1, 4e-6, _magnitude(r.array) + 1e-30)

    def c3(self, x, bound):
        """C3: 31-entry table, 31 integer + 31 float bins.  Bound 31: the mask is implied by the bin count (the
        assembler's peephole); 30: it is not."""
        tab = np.float32(0.5) + np.arange(31, dtype=np.float32) / np.float32(30)
        table = self.upload(Float32, tab)
        bins = self.upload(UInt32, np.zeros(31, np.uint32))
        hist = self.upload(Float32, np.zeros(31, np.float32))
        eight = Float32(8.0)
        k31 = Float32(31.0)
        idx = UInt32((x[0] - -4.0) * k31 / eight)
        del eight, k31
        mask = idx < bound
        w = ek.gather(Float32, table, idx, mask)
        ek.scatter_add(bins, UInt32(1), idx, mask)
        ek.scatter_add(hist, w, idx, mask)
        del idx, mask, w
        self.evaluate()
        self.keep("c3.bins" if bound == 31 else "c3m.bins", bins)
        self.keep("c3.hist" if bound == 31 else "c3m.hist", hist, 1)

    def global_gather_scatter(self, rng, n, x):
        """Global gather / scatter / scatter_add (targets too large for shared memory), masked."""
        x0, x1, x2, x3 = x
        m = 6000
        src = rng.uniforms(-1, 1, m)
        hi = rng.take(n) % np.uint32(m + 50)                   # some out of range: masked off
        S = self.upload(Float32, src)
        IDX = self.upload(UInt32, hi)
        TU = self.upload(UInt32, np.zeros(m, np.uint32))
        TF = self.upload(Float32, np.zeros(m, np.float32))
        ok = IDX < m
        g = ek.gather(Float32, S, IDX, ok)
        self.keep("gs.gather", g * x1)
        ek.scatter_add(TU, IDX & 7, IDX, ok)
        ek.scatter_add(TF, x2, IDX, ok)
        self.evaluate()
        self.keep("gs.add_u32", TU)
        self.keep("gs.add_f32", TF, 1)
        # plain scatter of a permutation (no conflicts: order-independent)
        perm = ((np.arange(n, dtype=np.uint64) * 7919 + 13) % n).astype(np.uint32)
        if len(np.unique(perm)) == n:
            P = self.upload(UInt32, perm)
            T2 = self.upload(Float32, np.zeros(n, np.float32))
            true = Mask(True)
            ek.scatter(T2, x0 + x3, P, true)
            del true
            self.evaluate()
            self.keep("gs.scatter", T2)

    def masks(self, x):
        """Mask arrays as outputs (8-bit stores) and as staged inputs (8-bit loads) of a later sweep; counts."""
        x0, x1, x2, x3 = x
        m1 = x0 > x1
        m2 = x2 <= 0.5
        not_m1 = ~m1
        m = (m1 & m2) | not_m1
        del not_m1
        self.keep("mask.out", m)
        self.keep("mask.select", ek.select(m, x0, x1 * 2.0))     # m now has storage: staged as bytes
        self.keep("mask.count", _op(UInt32, "COUNT", m))
        self.keep("mask.any", _op(Mask, "ANY", m2))
        self.keep("mask.all", _op(Mask, "ALL", m2))

    def integers(self, n, x):
        """Index arithmetic with literals, signed operations, conversions with rounding modes, and the remaining 32-bit
        operations of the fast kernel's set: integer multiply-add, signed / unsigned min, shifts by an array, every
        comparison, NOT, float rounding modes."""
        x0, x1, x2, x3 = x
        i = UInt32.arange(n)
        c = UInt32(974711)
        h = i * 2654435761 + c
        c = UInt32(2246822519)
        h = (h ^ (h >> 15)) * c
        del c
        self.keep("int.hash", h)
        s = Int32(x0 * 1000.0)
        t = -abs(s)
        self.keep("int.signed", ek.max_(s >> 3, t))
        del t
        self.keep("int.floor2int", ek.floor2int(Int32, x1))
        self.keep("int.ceil2int", ek.ceil2int(Int32, x1))
        t = Float32(h)
        self.keep("int.tofloat", Float32(s) + t)
        del t
        self.keep("int.lt", s < 0)
        u2 = h & 31
        self.keep("int.mad", ek.fmadd(h, u2, i))
        self.keep("int.minmax", ek.min_(s, 100 - s))
        t = s >> (s & 7)
        self.keep("int.shifts", (h << u2) ^ t)
        del t
        self.keep("int.not", ~h)
        t = x2.neq_(x3)
        right = (x0 <= x1) & t
        t = s >= 5
        left = h.neq_(i) | t
        del t
        cmp = left | right
        del left, right
        self.keep("cmp.mix", cmp ^ (h > 0x80000000))
        t = ek.trunc(x1 * 2.7)
        self.keep("f32.round", ek.round_(x0 * 3.3) + t)
        t = ek.floor(x1)
        self.keep("f32.eq", ek.select(ek.floor(x0).eq_(t), x2, x3))

    def reductions(self, x):
        """min / max / prod, a reduction reused by a wide consumer (second phase), the tape's guarded multiply-adds."""
        x0, x1, x2, x3 = x
        self.keep("red.hmin", _op(Float32, "HMIN", x0 * x1))
        self.keep("red.hmax", _op(Float32, "HMAX", ek.sin(x2)))
        one = Float32(1.0)
        self.keep("red.hprod", _op(Float32, "HPROD", ek.fmadd(x3, Float32(1e-4), one)), 1, 2e-3)
        del one
        sq = x0 * x0
        self.keep("red.normalised", sq / _op(Float32, "HSUM", sq), 1)
        t = ek.mul_nz(x2, ek.floor(x3))
        self.keep("red.mulnz", ek.fma_nz(x0, ek.floor(x1), t))
        t = ek.rsqrt(abs(x1))
        self.keep("red.rcp", ek.rcp(x0) + t)


def _dag_node(rng, fl, it):
    """One random node over the float values `fl` and the u32 values `it`."""
    kind = rng.below(22)
    a, b, c = (fl[rng.below(len(fl))] for _ in range(3))
    i, j = (it[rng.below(len(it))] for _ in range(2))
    if kind == 0:
        fl.append(a + b)
    elif kind == 1:
        fl.append(a - b)
    elif kind == 2:
        fl.append(a * b)
    elif kind == 3:
        fl.append(ek.fmadd(a, b, c))
    elif kind == 4:
        fl.append(ek.max_(a, b) if rng.below(2) else ek.min_(a, b))
    elif kind == 5:
        fl.append(abs(a))
    elif kind == 6:
        fl.append(-a)
    elif kind == 7:
        fl.append(ek.sqrt(abs(a)))
    elif kind == 8:
        fl.append(ek.floor(a) if rng.below(2) else ek.ceil(a))
    elif kind == 9:
        fl.append((ek.sin, ek.exp, ek.cos, ek.log)[rng.below(4)](a))
    elif kind == 10:
        fl.append(ek.select(a < b, a, c))
    elif kind == 11:
        it.append(i + j)
    elif kind == 12:
        it.append(i * j)
    elif kind == 13:
        t = i & j
        it.append((i ^ j) | t)
    elif kind == 14:
        s = 1 + rng.below(30)
        t = j >> s
        it.append((i << s) | t)
    elif kind == 15:
        it.append(ek.select(i < j, i, j))
    elif kind == 16:
        big = Float32(1.0e6)
        it.append(UInt32(ek.min_(abs(a), big)))
        fl.append(Float32(i >> 8))
    # literal operands in every position (the broadcast path)
    elif kind == 17:
        fl.append(ek.fmadd(a, Float32(rng.uniform(-2, 2)), b))
    elif kind == 18:
        fl.append(ek.fmadd(a, b, Float32(rng.uniform(-2, 2))))
    elif kind == 19:
        lit = Float32(rng.uniform(1, 3))
        fl.append(lit - a if rng.below(2) else lit / a)
    elif kind == 20:
        lit = Float32(1.5)
        fl.append(ek.select(a >= 0.25, lit, b))
    else:
        t = ek.min_(j, 77)
        it.append(ek.max_(i, 1000) - t)


def battery(upload, evaluate):
    b = _Battery(upload, evaluate)
    sizes = (4097, 100_003, (1 << 20) + 5)
    for seed in range(18):
        b.random_dag(seed, sizes[seed % 3])
    b.directed(100_003)
    b.directed((1 << 21) + 3)
    return b.records
