"""numpy interpreter of the sweep ISA (enoki_b200/csrc/ek_isa.h) for the CPU test-suite: executes the programs that the
planner + assembler produce (`enoki_b200.debug_program()`), so that scheduling, slot allocation, superinstruction
fusion, reduction phases and operand encoding are checked on machines without a GPU.  TEST INFRASTRUCTURE: it mirrors
what ek_sweep.cu does per element (32- and 64-bit value types, the latter as lo/hi planes exactly like the kernel;
32-bit gathers / scatters incl. the shared-memory table / privatised-bin helpers; float scatter_add is accumulated in
element order, so compare it with a tolerance) and uses the C oracle for the operations numpy cannot round identically (fma, Cephes)."""
import ctypes

import numpy as np

F_ST, F_R64, F_HAS_B, F_HAS_C, F_B64, F_C64, F_A64, F_HAS_A, F_NEG_A, F_ABS_A, F_STG, F_RACC = 1, 2, 4, 8, 0x10, 0x20, 0x40, 0x80, 0x100, 0x200, 0x400, 0x4000
OP_NONE = 0xFFFF
NEG_ZERO = 0x80000000                      # bits of -0.0f, the start value of float scatter_add bins
SZ = ctypes.c_size_t
T_FLOAT32, T_INT32, T_UINT32, T_BOOL, T_INT64, T_UINT64, T_FLOAT64 = 10, 5, 6, 12, 7, 8, 11


class Unsupported(Exception):
    pass


def _P(a):
    return a.ctypes.data_as(ctypes.c_void_p)


FF_B, FF_C, FF_BU, FF_CU, FF_ST, FF_STG, FF_RACC, FF_VU, FF_MU = 1, 2, 4, 8, 0x10, 0x20, 0x40, 0x80, 0x100


def raise_fast(fast, fop_names, op_index):
    """The lowered program of the 32-bit fast kernel (ek_isa.h "lowered instruction format", produced by lower_fast in
    ek_eval.cpp) translated back into (op, flags, dst, b, c, a, imm) tuples of the assembler's form, so that the same
    per-element interpreter executes it: checks the splitting of accumulator loads / modifiers, the _U twins, the
    operand encoding against the fast kernel's shared-memory layout and the post-action flags on the CPU."""
    T, off_slots, n_tmp = fast["T"], fast["off_slots"], fast["n_tmp"]
    slot_bytes = T * 16 * 4

    def slot(off16):                                # byte offset >> 4 -> temporary slot / staged unit code
        q, r = divmod((off16 << 4) - off_slots, slot_bytes)
        assert r == 0 and q >= 0, ("operand offset is not a slot boundary", off16)
        return q if q < n_tmp else 0x4000 | (q - n_tmp)

    def uni(i):
        return 0x8000 | i

    def conv(t):
        fop, fl, b, c, dst, aux, imm = t
        name = fop_names[fop]
        flags, cb, cc, ca, d = 0, OP_NONE, OP_NONE, OP_NONE, 0
        if fl & FF_B: flags |= F_HAS_B; cb = slot(b)
        if fl & FF_BU: flags |= F_HAS_B; cb = uni(b)
        if fl & FF_C: flags |= F_HAS_C; cc = slot(c)
        if fl & FF_CU: flags |= F_HAS_C; cc = uni(c)
        if name in ("LOAD", "LOADU"):
            flags |= F_HAS_B; cb = slot(b) if name == "LOAD" else uni(b); name = "LOAD_32"
        elif name in ("EXPN_F32", "SQRTA_F32"):
            flags |= F_NEG_A if name == "EXPN_F32" else F_ABS_A
            name = "EXP_F32" if name == "EXPN_F32" else "SQRT_F32"
        elif name.endswith("_U") and name[:-2] in op_index:
            flags |= F_HAS_B; cb = uni(b); name = name[:-2]
        elif name == "FMA_F32_UB": flags |= F_HAS_B; cb = uni(b); name = "FMA_F32"
        elif name == "FMA_F32_UC": flags |= F_HAS_C; cc = uni(c); name = "FMA_F32"
        elif name == "FMAC_F32_UB": flags |= F_HAS_B; cb = uni(b); name = "FMAC_F32"
        elif name in ("LD_U8", "LD_S8"): cb = slot(b)
        elif name.startswith("GATHER"):
            if fl & FF_MU: flags |= F_HAS_B; cb = uni(b)
        elif name.startswith("SCATTER"):
            if fl & FF_VU: flags |= F_HAS_B; cb = uni(b)
            if fl & FF_MU: flags |= F_HAS_C; cc = uni(c)
        elif name == "RFIN":
            flags |= F_HAS_B; cb = slot(b); d = dst
        elif name == "SMEM_ZERO":
            d = dst
        if fl & FF_ST: flags |= F_ST; d = slot(dst)
        if fl & FF_STG: flags |= F_STG
        if fl & FF_RACC:
            d = slot(dst)
            if name == "RACC": imm = aux
            else: flags |= F_RACC; ca = aux
        return [op_index[name], flags, d, cb, cc, ca, imm]

    return {k: [conv(t) for t in fast[k]] for k in ("init", "body", "fini")}


def _f2ll(x, mode, unsigned):
    """float / double -> int64 (uint64) of the kernel: values outside [-2^63, 2^63) (for uint64 [-2^63, 2^64)) and NaN
    give 0x8000000000000000, the rest is rounded in `mode` and wraps to 64 bits."""
    r = {0: np.trunc, 1: np.floor, 2: np.ceil, 3: np.rint}[mode](x)
    ok = (x >= -9.2233720368547758e18) & (x < 9.2233720368547758e18)
    v = np.where(ok, np.where(ok, r, 0).astype(np.int64), np.int64(-9223372036854775808)).view(np.uint64)
    if unsigned:
        top = (x >= 9.2233720368547758e18) & (x < 1.8446744073709552e19)
        v = np.where(top, (np.where(top, x, 0) - 9.2233720368547758e18).astype(np.int64).view(np.uint64) + np.uint64(1 << 63), v)
    return v


def _int64_ops(base, signed, ua, ub):
    """64-bit mulhi, div / mod (ek_div64: /0 and INT64_MIN / -1 as the kernel guards them) and bit counts, in Python
    integers."""
    M = (1 << 64) - 1
    sv = lambda v: v - (1 << 64) if signed and v >> 63 else v
    out = []
    for k in range(len(ua)):
        a = int(ua[k]); b = int(ub[k]) if ub is not None else 0
        if base in ("DIVR", "MODR"):
            a, b = b, a
        a, b = sv(a), sv(b)
        if base == "MULHI": r = (a * b) >> 64
        elif base == "POPC": r = bin(a & M).count("1")
        elif base == "CLZ": r = 64 - (a & M).bit_length()
        elif base == "CTZ": r = ((a & -a) & M).bit_length() - 1 if a & M else 64
        elif base.startswith("DIV"):
            if b == 0: r = 0 if signed else M
            elif b == -1 and signed: r = -a
            else:
                q = abs(a) // abs(b); r = q if (a < 0) == (b < 0) else -q
        else:
            if b == 0: r = 0 if signed else a
            elif b == -1 and signed: r = 0
            else:
                q = abs(a) // abs(b); r = a - (q if (a < 0) == (b < 0) else -q) * b
        out.append(r & M)
    return np.array(out, np.uint64)


class Emulator:
    prefer_fast = False        # execute the lowered fast-kernel program of a sweep when the dump carries one

    def __init__(self, oracle, arrays, by_address=None):
        """arrays: variable index -> numpy array (data of evaluated inputs); by_address: device address -> variable index
        (gather sources / scatter targets reach the program as raw pointers, not as variables)."""
        self.oracle = oracle
        self.vars = {k: np.ascontiguousarray(v) for k, v in arrays.items()}
        self.by_address = dict(by_address or {})

    # ---- helpers
    @staticmethod
    def _f(x): return x.view(np.float32)
    @staticmethod
    def _u(x): return np.ascontiguousarray(x).view(np.uint32)

    def _unary(self, which, x):
        xf = np.ascontiguousarray(self._f(x)); out = np.zeros_like(xf)
        self.oracle.or_unary_f32(which, _P(xf), _P(out), SZ(len(xf)))
        return self._u(out)

    def _fma(self, a, b, c):
        a, b, c = (np.ascontiguousarray(self._f(v)) for v in (a, b, c)); out = np.zeros_like(a)
        self.oracle.or_fma_f32(_P(a), _P(b), _P(c), _P(out), SZ(len(a)))
        return self._u(out)

    def _minmax(self, is_max, a, b):
        a, b = (np.ascontiguousarray(self._f(v)) for v in (a, b)); out = np.zeros_like(a)
        self.oracle.or_minmax_f32(int(is_max), _P(a), _P(b), _P(out), SZ(len(a)))
        return self._u(out)

    # ---- 64-bit values as (lo, hi) planes
    @staticmethod
    def _j(lo, hi): return (hi.astype(np.uint64) << np.uint64(32)) | lo.astype(np.uint64)
    @staticmethod
    def _s(v):
        v = np.ascontiguousarray(v).view(np.uint64)
        return (v & np.uint64(0xffffffff)).astype(np.uint32), (v >> np.uint64(32)).astype(np.uint32)

    def _unary64(self, which, x):
        xf = np.ascontiguousarray(x.view(np.float64)); out = np.zeros_like(xf)
        self.oracle.or_unary_f64(which, _P(xf), _P(out), SZ(len(xf)))
        return out

    def _exec64(self, name, imm, R, Rh, B, Bh, C, Ch, staged, cb):
        """64-bit and width-changing operations; returns (lo, hi), "store", "ldg", or None if `name` is a 32-bit op."""
        J, S = self._j, self._s
        u = lambda lo, hi: J(lo, hi)
        i = lambda lo, hi: J(lo, hi).view(np.int64)
        d = lambda lo, hi: J(lo, hi).view(np.float64)
        with np.errstate(all="ignore"):
            if name == "LD_64": return S(staged[cb & 0x3fff])
            if name == "LDG_64": return "ldg"
            if name == "ST_64": return "store"
            if name.endswith("_F64") and not name.startswith("CVT_"):
                a = d(R, Rh); b = d(B, Bh) if Bh is not None else None; c = d(C, Ch) if Ch is not None else None
                base = name[:-4]
                if base in ("FMA", "FMAC", "FMANZ", "FMANZC"):
                    x, y, z = (a, b, c) if base in ("FMA", "FMANZ") else (b, c, a)
                    x, y, z = (np.ascontiguousarray(v) for v in (x, y, z)); out = np.zeros_like(x)
                    self.oracle.or_fma_f64(_P(x), _P(y), _P(z), _P(out), SZ(len(x)))
                    if base.startswith("FMANZ"):                      # a zero factor gives the addend as it is
                        out = np.where((x == 0) | (y == 0), z, out)
                    return S(out)
                if base in ("MIN", "MAX", "MINR", "MAXR"):
                    x, y = (a, b) if len(base) == 3 else (b, a)
                    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y); out = np.zeros_like(x)
                    self.oracle.or_minmax_f64(int(base.startswith("MAX")), _P(x), _P(y), _P(out), SZ(len(x)))
                    return S(out)
                if base in ("LT", "LE", "GT", "GE", "EQ", "NE"):
                    fn = {"LT": np.less, "LE": np.less_equal, "GT": np.greater, "GE": np.greater_equal, "EQ": np.equal, "NE": np.not_equal}[base]
                    return fn(a, b).astype(np.uint32), Rh
                r = {"ADD": lambda: a + b, "SUB": lambda: a - b, "SUBR": lambda: b - a, "MUL": lambda: a * b, "DIV": lambda: a / b,
                     "DIVR": lambda: b / a, "ABS": lambda: np.abs(a), "NEG": lambda: -a, "SQRT": lambda: np.sqrt(a),
                     "FLOOR": lambda: np.floor(a), "CEIL": lambda: np.ceil(a), "ROUND": lambda: np.rint(a), "TRUNC": lambda: np.trunc(a),
                     "RCP": lambda: 1.0 / a, "RSQRT": lambda: 1.0 / np.sqrt(a),
                     "MULNZ": lambda: np.where((a == 0) | (b == 0), 0.0, a * b),
                     "EXP": lambda: self._unary64(2, a), "LOG": lambda: self._unary64(3, a), "SIN": lambda: self._unary64(0, a),
                     "COS": lambda: self._unary64(1, a)}.get(base)
                if r is None:
                    raise Unsupported(name)
                return S(np.ascontiguousarray(r()))
            if name.endswith(("_I64", "_U64", "_64")) and not name.startswith("CVT_"):
                signed = name.endswith("_I64")
                a = i(R, Rh) if signed else u(R, Rh)
                b = (i(B, Bh) if signed else u(B, Bh)) if Bh is not None else None
                base = name.rsplit("_", 1)[0]
                if base in ("SHL", "SHR"):                              # the count is the 32-bit low plane only
                    cnt = B.astype(np.uint64)
                    if base == "SHL": return S(np.where(cnt >= 64, np.uint64(0), u(R, Rh) << (cnt & np.uint64(63))))
                    if signed: return S((i(R, Rh) >> np.minimum(cnt, np.uint64(63)).astype(np.int64)).view(np.uint64))
                    return S(np.where(cnt >= 64, np.uint64(0), u(R, Rh) >> (cnt & np.uint64(63))))
                if base in ("SHLR", "SHRR"):
                    val = i(B, Bh) if signed else u(B, Bh); cnt = R.astype(np.uint64)
                    if base == "SHLR": return S(np.where(cnt >= 64, np.uint64(0), u(B, Bh) << (cnt & np.uint64(63))))
                    if signed: return S((val >> np.minimum(cnt, np.uint64(63)).astype(np.int64)).view(np.uint64))
                    return S(np.where(cnt >= 64, np.uint64(0), val >> (cnt & np.uint64(63))))
                if base in ("LT", "LE", "GT", "GE"):
                    fn = {"LT": np.less, "LE": np.less_equal, "GT": np.greater, "GE": np.greater_equal}[base]
                    return fn(a, b).astype(np.uint32), Rh
                if base == "EQ": return (u(R, Rh) == u(B, Bh)).astype(np.uint32), Rh
                if base == "NE": return (u(R, Rh) != u(B, Bh)).astype(np.uint32), Rh
                if base == "SEL_M": return np.where(R != 0, B, C), np.where(R != 0, Bh, Ch)
                if base == "SEL_T": return np.where(B != 0, R, C), np.where(B != 0, Rh, Ch)
                if base == "SEL_F": return np.where(B != 0, C, R), np.where(B != 0, Ch, Rh)
                if base == "LOAD": return B, Bh
                ua, ub = u(R, Rh), (u(B, Bh) if Bh is not None else None)
                if base in ("MULHI", "DIV", "DIVR", "MOD", "MODR", "POPC", "CLZ", "CTZ"):
                    return S(_int64_ops(base, signed, ua, ub))
                r = {"ADD": lambda: ua + ub, "SUB": lambda: ua - ub, "SUBR": lambda: ub - ua, "MUL": lambda: ua * ub,
                     "MAD": lambda: ua * ub + u(C, Ch), "MADC": lambda: ub * u(C, Ch) + ua,
                     "MIN": lambda: np.minimum(a, b).view(np.uint64), "MAX": lambda: np.maximum(a, b).view(np.uint64),
                     "ABS": lambda: np.where(i(R, Rh) < 0, np.uint64(0) - ua, ua), "NEG": lambda: np.uint64(0) - ua,
                     "NOT": lambda: ~ua, "AND": lambda: ua & ub, "OR": lambda: ua | ub, "XOR": lambda: ua ^ ub}.get(base)
                if r is None:
                    raise Unsupported(name)
                return S(np.ascontiguousarray(r()))
            if name.startswith("CVT_"):
                f32 = R.view(np.float32)
                if name == "CVT_I32_I64": return R, (R.view(np.int32) >> 31).view(np.uint32)
                if name == "CVT_U32_U64": return R, np.zeros_like(R)
                if name == "CVT_64_32": return R, Rh
                if name == "CVT_F32_F64": return S(f32.astype(np.float64))
                if name == "CVT_F64_F32": return d(R, Rh).astype(np.float32).view(np.uint32), Rh
                if name == "CVT_I32_F64": return S(R.view(np.int32).astype(np.float64))
                if name == "CVT_U32_F64": return S(R.astype(np.float64))
                if name == "CVT_I64_F64": return S(i(R, Rh).astype(np.float64))
                if name == "CVT_U64_F64": return S(u(R, Rh).astype(np.float64))
                if name == "CVT_I64_F32": return i(R, Rh).astype(np.float32).view(np.uint32), Rh
                if name == "CVT_U64_F32": return u(R, Rh).astype(np.float32).view(np.uint32), Rh
                if name in ("CVT_F64_I64", "CVT_F64_U64", "CVT_F32_I64", "CVT_F32_U64"):
                    x = d(R, Rh) if "F64" in name else f32.astype(np.float64)
                    return S(_f2ll(x, imm, name.endswith("U64")))
                if name in ("CVT_F64_I32",):                     # cvttpd2dq of the rounded value
                    r = {0: np.trunc, 1: np.floor, 2: np.ceil, 3: np.rint}[imm](d(R, Rh))
                    ok = (r >= -2147483648.0) & (r < 2147483648.0)
                    return np.where(ok, np.where(ok, r, 0).astype(np.int64), np.int64(-2147483648)).astype(np.int32).view(np.uint32), Rh
                if name == "CVT_F64_U32":                         # the low word of the int64 conversion
                    return (_f2ll(d(R, Rh), imm, False) & np.uint64(0xffffffff)).astype(np.uint32), Rh
                return None                                       # 32-bit conversions are handled by the caller
        return None

    def run(self, program):
        names = program["ops"]
        self.fast_sweeps = 0
        for sw in program["sweeps"]:
            if self.prefer_fast and "fast" in sw:
                raised = raise_fast(sw["fast"], program["fops"], {n: i for i, n in enumerate(names)})
                sw = dict(sw, **raised)
                self.fast_sweeps += 1
            self._sweep(names, sw)

    def _sweep(self, names, sw):
        n = sw["n"]
        lits, argw = sw["lits"], list(sw["argw"])
        n_lit, n_arg = len(lits), len(argw)
        ptr = {}                                    # argw index -> variable
        for aw, var, _out, address in sw["ptr_fix"]:
            ptr[aw] = self.by_address.get(address, var) if var not in self.vars else var
        # uniform pool = literals | argument words | scalar (lo, hi) pairs
        uni = [np.uint32(v) for v in lits] + [None] * n_arg
        for var, typ in sw["scalars"]:
            v = self.vars[var]
            if v.dtype.itemsize == 8:
                bits = int(v.reshape(-1).view(np.uint64)[0])
                uni += [np.uint32(bits & 0xffffffff), np.uint32(bits >> 32)]
                continue
            lo = np.uint32(1 if (typ == T_BOOL and v.reshape(-1)[0]) else v.reshape(-1).view(np.uint32 if v.dtype.itemsize == 4 else v.dtype)[0])
            uni += [lo, np.uint32(0)]
        staged = {}
        for var, unit, es in sw["staged"]:
            a = self.vars[var]
            assert a.size == n, (var, a.size, n)
            if es == 4:
                staged[unit] = self._u(a)
            elif es == 8:
                staged[unit] = np.ascontiguousarray(a).view(np.uint64)        # unpacked by LD_64
            elif es == 1:
                staged[unit] = np.ascontiguousarray(a).view(np.uint8)         # unpacked by LD_U8 / LD_S8
            elif es == 2:
                staged[unit] = np.ascontiguousarray(a).view(np.uint16)        # unpacked by LD_U16 / LD_S16
            else:
                raise Unsupported("staged input of element size %d" % es)
        out_type = {var: typ for var, _aw, _bytes, typ in sw["outputs"]}
        slots = {}
        smem = {}                                   # descriptor uniform index -> staged table / privatised bins
        state = {"R": np.zeros(n, np.uint32), "Rh": np.zeros(n, np.uint32)}

        def desc(ui):                               # {smem_off, count, copies, uniform index of the pointer}
            di = ui - n_lit
            return argw[di + 1], ptr[argw[di + 3] - n_lit]

        def gs_target(imm):                         # global gather / scatter: imm = uniform | stride << 16 | signed << 31
            var = var_of_uniform(imm & 0xffff)
            stride = (imm >> 16) & 0x7fff
            if stride != 4:
                raise Unsupported("gather/scatter stride %d" % stride)
            return var

        idx = np.arange(n, dtype=np.uint32)

        def bcast(v):
            return np.full(n, v, np.uint32)

        def fetch(code):
            if code == OP_NONE:
                raise AssertionError("fetch of an absent operand")
            if (code & 0xC000) == 0xC000:
                raise Unsupported("global operand")
            if code & 0x8000:
                v = uni[code & 0x3fff]
                if v is None:
                    raise AssertionError("argument word used as a value")
                return bcast(v)
            if code & 0x4000:
                return staged[code & 0x3fff].copy()
            if code not in slots:
                raise AssertionError("read of slot %d before it was written" % code)
            return slots[code].copy()

        def fetch_hi(code):
            if code & 0x8000:
                return bcast(uni[(code & 0x3fff) + 1])
            if code & 0x4000:
                raise AssertionError("high plane of a staged operand")
            if code + 1 not in slots:
                raise AssertionError("read of the high plane of slot %d before it was written" % code)
            return slots[code + 1].copy()

        def var_of_uniform(ui):
            aw = ui - n_lit
            assert 0 <= aw < n_arg and aw in ptr, ("uniform index is not a pointer argument", ui)
            return ptr[aw]

        def store_var(var, R):
            typ = out_type.get(var, T_UINT32)
            if typ == T_BOOL:
                self.vars[var] = (R & 1).astype(np.bool_)
            elif typ == T_FLOAT32:
                self.vars[var] = R.view(np.float32).copy()
            elif typ == T_INT32:
                self.vars[var] = R.view(np.int32).copy()
            elif typ == T_UINT32:
                self.vars[var] = R.copy()
            elif typ in (T_INT64, T_UINT64, T_FLOAT64):
                v = self._j(R, state["Rh"])
                self.vars[var] = v.view({T_INT64: np.int64, T_UINT64: np.uint64, T_FLOAT64: np.float64}[typ]).copy()
            else:
                raise Unsupported("output type %d" % typ)

        def racc(slot, kc):
            kind, cls = kc & 0xff, (kc >> 8) & 0xff
            acc = slots[slot]
            R = state["R"]
            with np.errstate(all="ignore"):
                if cls == 0:
                    a, r = self._f(acc), self._f(R)
                    res = {0: a + r, 1: a * r}.get(kind)
                    if res is None:
                        res = self._f(self._minmax(kind == 3, R, acc))       # red_combine: min_x86(y, x)
                elif cls in (1, 2):
                    a = acc.view(np.int32 if cls == 1 else np.uint32); r = R.view(a.dtype)
                    res = {0: a + r, 1: a * r, 2: np.minimum(a, r), 3: np.maximum(a, r)}[kind]
                else:                                   # F64 / I64 / U64: (lo, hi) planes in slots dst, dst + 1
                    a, r = self._j(acc, slots[slot + 1]), self._j(R, state["Rh"])
                    if cls == 3 and kind >= 2:          # red_combine: min_x86(y, x)
                        x, y = np.ascontiguousarray(r.view(np.float64)), np.ascontiguousarray(a.view(np.float64))
                        res = np.zeros_like(x)
                        self.oracle.or_minmax_f64(int(kind == 3), _P(x), _P(y), _P(res), SZ(len(x)))
                    elif cls == 3:
                        a, r = a.view(np.float64), r.view(np.float64)
                        res = a + r if kind == 0 else a * r
                    elif kind <= 1:
                        res = a + r if kind == 0 else a * r
                    else:
                        dt = np.int64 if cls == 4 else np.uint64
                        res = (np.minimum if kind == 2 else np.maximum)(a.view(dt), r.view(dt))
                    slots[slot], slots[slot + 1] = self._s(res)
                    return
            slots[slot] = self._u(np.ascontiguousarray(res))

        def rfin(B, Bh, imm, dst):
            kind, cls = imm & 0xff, (imm >> 8) & 0xff
            if cls > 2:
                x = self._j(B, Bh)
                if cls == 3:
                    x = x.view(np.float64)
                    val = np.array([{0: x.sum(), 1: np.prod(x), 2: x.min(), 3: x.max()}[kind]], np.float64)
                else:
                    dt = np.int64 if cls == 4 else np.uint64
                    r = {0: lambda: np.sum(x, dtype=np.uint64), 1: lambda: np.multiply.reduce(x),
                         2: lambda: x.view(dt).min(), 3: lambda: x.view(dt).max()}[kind]()
                    val = np.array([r]).astype(dt)
                self.vars[var_of_uniform(dst)] = val
                return
            if cls == 0:
                x = self._f(B).astype(np.float64)
                r = {0: x.sum(), 1: np.prod(x), 2: x.min(), 3: x.max()}[kind]
                val = np.array([r], np.float32)
            else:
                dt = np.int32 if cls == 1 else np.uint32
                x = B.view(dt)
                if kind == 0: r = dt(int(x.astype(np.int64).sum()) & 0xffffffff) if dt is np.uint32 else np.int64(x.astype(np.int64).sum()).astype(np.int32)
                elif kind == 1:
                    acc = 1
                    for v in x.tolist(): acc = (acc * v) & 0xffffffff
                    r = np.uint32(acc).astype(dt) if dt is np.uint32 else np.uint32(acc).view(np.int32)
                else: r = x.min() if kind == 2 else x.max()
                val = np.array([r]).astype(dt)
            self.vars[var_of_uniform(dst)] = val

        def execute(ins):
            op, flags, dst, cb, cc, ca, imm = ins
            name = names[op]
            if flags & F_HAS_A:
                state["R"] = fetch(ca)
                if flags & F_A64:
                    state["Rh"] = fetch_hi(ca)
            if flags & F_ABS_A:
                state["R"] = state["R"] & np.uint32(0x7fffffff)
            if flags & F_NEG_A:
                state["R"] = state["R"] ^ np.uint32(0x80000000)
            R = state["R"]
            B = fetch(cb) if flags & F_HAS_B else None
            C = fetch(cc) if flags & F_HAS_C else None
            Bh = fetch_hi(cb) if flags & F_B64 else None
            Ch = fetch_hi(cc) if flags & F_C64 else None
            Rh = state["Rh"]
            f = self._f
            if name.endswith(("_F64", "_I64", "_U64", "_64")) or name.startswith(("CVT_", "LD_64", "LDG_64", "ST_64")):
                handled = self._exec64(name, imm, R, Rh, B, Bh, C, Ch, staged, cb)
                if handled is not None:
                    if handled == "store":
                        store_var(var_of_uniform(imm), R); return
                    if handled == "ldg":
                        v = np.ascontiguousarray(self.vars[var_of_uniform(imm)]).view(np.uint64)
                        state["R"], state["Rh"] = self._s(v)
                    else:
                        state["R"], state["Rh"] = handled
                    if flags & F_RACC:
                        racc(dst, ca)
                    if flags & F_STG:
                        store_var(var_of_uniform(imm), state["R"])
                    if flags & F_ST:
                        slots[dst] = state["R"].copy()
                        if flags & F_R64:
                            slots[dst + 1] = state["Rh"].copy()
                    return
            with np.errstate(all="ignore"):
                if name == "NOP": pass
                elif name == "ADD_F32": R = self._u(f(R) + f(B))
                elif name == "SUB_F32": R = self._u(f(R) - f(B))
                elif name == "SUBR_F32": R = self._u(f(B) - f(R))
                elif name == "MUL_F32": R = self._u(f(R) * f(B))
                elif name == "DIV_F32": R = self._u(f(R) / f(B))
                elif name == "DIVR_F32": R = self._u(f(B) / f(R))
                elif name == "FMA_F32": R = self._fma(R, B, C)
                elif name == "FMAC_F32": R = self._fma(B, C, R)
                elif name == "MULNZ_F32": R = np.where((f(R) == 0) | (f(B) == 0), np.uint32(0), self._u(f(R) * f(B)))
                elif name == "FMANZ_F32": R = np.where((f(R) == 0) | (f(B) == 0), C, self._fma(R, B, C))
                elif name == "FMANZC_F32": R = np.where((f(B) == 0) | (f(C) == 0), R, self._fma(B, C, R))
                elif name in ("MIN_F32", "MAX_F32"): R = self._minmax(name == "MAX_F32", R, B)
                elif name in ("MINR_F32", "MAXR_F32"): R = self._minmax(name == "MAXR_F32", B, R)
                elif name == "ABS_F32": R = R & np.uint32(0x7fffffff)
                elif name == "NEG_F32": R = R ^ np.uint32(0x80000000)
                elif name == "SQRT_F32": R = self._u(np.sqrt(f(R)))
                elif name == "RCP_F32": R = self._u(np.float32(1.0) / f(R))                      # correctly rounded 1/x (DESIGN.md 4)
                elif name == "RSQRT_F32": R = self._u(np.float32(1.0) / np.sqrt(f(R)))
                elif name == "EXP_F32": R = self._unary(2, R)
                elif name == "LOG_F32": R = self._unary(3, R)
                elif name == "SIN_F32": R = self._unary(0, R)
                elif name == "COS_F32": R = self._unary(1, R)
                elif name == "FLOOR_F32": R = self._u(np.floor(f(R)))
                elif name == "CEIL_F32": R = self._u(np.ceil(f(R)))
                elif name == "ROUND_F32": R = self._u(np.rint(f(R)))
                elif name == "TRUNC_F32": R = self._u(np.trunc(f(R)))
                elif name in ("LT_F32", "LE_F32", "GT_F32", "GE_F32", "EQ_F32", "NE_F32"):
                    fn = {"LT": np.less, "LE": np.less_equal, "GT": np.greater, "GE": np.greater_equal, "EQ": np.equal, "NE": np.not_equal}[name[:2]]
                    R = fn(f(R), f(B)).astype(np.uint32)
                elif name == "ADD_I32": R = R + B
                elif name == "SUB_I32": R = R - B
                elif name == "SUBR_I32": R = B - R
                elif name == "MUL_I32": R = R * B
                elif name == "MAD_I32": R = R * B + C
                elif name == "MADC_I32": R = B * C + R
                elif name == "NEG_I32": R = np.uint32(0) - R
                elif name == "ABS_I32": R = np.where(R.view(np.int32) < 0, np.uint32(0) - R, R)
                elif name == "MULHI_U32": R = ((R.astype(np.uint64) * B.astype(np.uint64)) >> np.uint64(32)).astype(np.uint32)
                elif name == "MULHI_I32": R = ((R.view(np.int32).astype(np.int64) * B.view(np.int32).astype(np.int64)) >> np.int64(32)).astype(np.int32).view(np.uint32)
                elif name in ("DIV_U32", "DIVR_U32", "MOD_U32", "MODR_U32"):
                    a, b = (R, B) if not name.startswith(("DIVR", "MODR")) else (B, R)
                    bz = b == 0
                    bs = np.where(bz, np.uint32(1), b)
                    R = np.where(bz, np.uint32(0xffffffff), a // bs) if name.startswith("DIV") else np.where(bz, a, a % bs)
                elif name in ("DIV_I32", "DIVR_I32", "MOD_I32", "MODR_I32"):
                    a, b = (R, B) if not name.startswith(("DIVR", "MODR")) else (B, R)
                    a = a.view(np.int32).astype(np.int64); b = b.view(np.int32).astype(np.int64)
                    bz = b == 0
                    bs = np.where(bz, 1, b)
                    q = np.sign(a) * np.sign(bs) * (np.abs(a) // np.abs(bs))          # C truncation
                    if name.startswith("DIV"):
                        R = np.where(bz, 0, q).astype(np.int64).astype(np.int32).view(np.uint32)   # (INT_MIN / -1 wraps)
                        R = np.where((b == -1), (np.uint32(0) - a.astype(np.int32).view(np.uint32)), R)
                    else:
                        R = np.where(bz | (b == -1), 0, a - q * bs).astype(np.int32).view(np.uint32)
                elif name == "POPC_32": R = np.array([bin(int(v)).count("1") for v in R], np.uint32) if len(R) < 200000 else (_ for _ in ()).throw(Unsupported("popc of a large array"))
                elif name == "CLZ_32": R = np.array([32 - int(v).bit_length() for v in R], np.uint32) if len(R) < 200000 else (_ for _ in ()).throw(Unsupported("clz of a large array"))
                elif name == "CTZ_32": R = np.array([(int(v) & -int(v)).bit_length() - 1 if v else 32 for v in R], np.uint32) if len(R) < 200000 else (_ for _ in ()).throw(Unsupported("ctz of a large array"))
                elif name == "SEXT8": R = R.astype(np.uint8).view(np.int8).astype(np.int32).view(np.uint32)
                elif name == "SEXT16": R = R.astype(np.uint16).view(np.int16).astype(np.int32).view(np.uint32)
                elif name == "ZEXT8": R = R & np.uint32(0xff)
                elif name == "ZEXT16": R = R & np.uint32(0xffff)
                elif name in ("LD_U8", "LD_S8"):
                    v = staged[cb & 0x3fff]
                    R = v.astype(np.uint32) if name == "LD_U8" else v.view(np.int8).astype(np.int32).view(np.uint32)
                elif name in ("LD_U16", "LD_S16"):
                    v = staged[cb & 0x3fff]
                    R = v.astype(np.uint32) if name == "LD_U16" else v.view(np.int16).astype(np.int32).view(np.uint32)
                elif name == "ST_8":
                    var = var_of_uniform(imm)
                    self.vars[var] = (R & 0xff).astype(np.uint8).view(np.bool_) if out_type.get(var) == T_BOOL else (R & 0xff).astype(np.uint8)
                    return
                elif name == "ST_16":
                    var = var_of_uniform(imm)
                    self.vars[var] = (R & 0xffff).astype(np.uint16)
                    return
                elif name == "NOT_32": R = ~R
                elif name == "AND_32": R = R & B
                elif name == "OR_32": R = R | B
                elif name == "XOR_32": R = R ^ B
                elif name == "SHL_32": R = np.where(B >= 32, np.uint32(0), R << (B & np.uint32(31)))
                elif name == "SHR_U32": R = np.where(B >= 32, np.uint32(0), R >> (B & np.uint32(31)))
                elif name == "SHR_I32": R = (R.view(np.int32) >> np.minimum(B, np.uint32(31)).astype(np.int32)).view(np.uint32)
                elif name in ("MIN_U32", "MAX_U32"): R = (np.minimum if name == "MIN_U32" else np.maximum)(R, B)
                elif name in ("MIN_I32", "MAX_I32"): R = (np.minimum if name == "MIN_I32" else np.maximum)(R.view(np.int32), B.view(np.int32)).view(np.uint32)
                elif name in ("LT_U32", "LE_U32", "GT_U32", "GE_U32"):
                    fn = {"LT": np.less, "LE": np.less_equal, "GT": np.greater, "GE": np.greater_equal}[name[:2]]
                    R = fn(R, B).astype(np.uint32)
                elif name in ("LT_I32", "LE_I32", "GT_I32", "GE_I32"):
                    fn = {"LT": np.less, "LE": np.less_equal, "GT": np.greater, "GE": np.greater_equal}[name[:2]]
                    R = fn(R.view(np.int32), B.view(np.int32)).astype(np.uint32)
                elif name == "EQ_32": R = (R == B).astype(np.uint32)
                elif name == "NE_32": R = (R != B).astype(np.uint32)
                elif name == "NOT_B": R = R ^ np.uint32(1)
                elif name == "NEZ_32": R = (R != 0).astype(np.uint32)
                elif name == "SEL_M_32": R = np.where(R != 0, B, C)
                elif name == "SEL_T_32": R = np.where(B != 0, R, C)
                elif name == "SEL_F_32": R = np.where(B != 0, C, R)
                elif name == "LOAD_32": R = B
                elif name == "INDEX": R = idx.copy()
                elif name == "CVT_F32_U32":
                    # the AVX2 sequence of the CPU path (array_avx2.h), after rounding:
                    # r >= 2^31 ? cvttps2dq(r - 2^31) + 2^31 : cvttps2dq(r), cvttps2dq giving 0x80000000 out of range
                    r = {0: np.trunc, 1: np.floor, 2: np.ceil, 3: np.rint}[imm](f(R)).astype(np.float64)
                    hi = r >= 2147483648.0
                    v = np.where(hi, r - 2147483648.0, r)
                    ok = (v >= -2147483648.0) & (v < 2147483648.0)
                    w = np.where(ok, np.where(ok, v, 0).astype(np.int64), np.int64(-2147483648)).astype(np.int32).view(np.uint32)
                    R = np.where(hi, w + np.uint32(0x80000000), w)
                elif name == "CVT_F32_I32":
                    x = f(R)
                    r = {0: np.trunc, 1: np.floor, 2: np.ceil, 3: np.rint}[imm](x)
                    ok = (x >= -2147483648.0) & (x < 2147483648.0)
                    R = np.where(ok, np.where(ok, r, 0).astype(np.int64), np.int64(-2147483648)).astype(np.int32).view(np.uint32)
                elif name == "CVT_I32_F32": R = self._u(R.view(np.int32).astype(np.float32))
                elif name == "CVT_U32_F32": R = self._u(R.astype(np.float32))
                elif name == "LDG_32": R = self._u(self.vars[var_of_uniform(imm)]).copy()
                elif name == "ST_32": store_var(var_of_uniform(imm), R)
                elif name == "SMEM_ZERO":                    # dst = 1: float bins, which start at -0.0
                    cnt, _var = desc(imm); smem[imm] = np.full(cnt, NEG_ZERO if dst else 0, np.uint32); return
                elif name == "SMEM_LOAD_TABLE":
                    cnt, var = desc(imm); smem[imm] = self._u(self.vars[var])[:cnt].copy(); return
                elif name in ("SMEM_FLUSH_ADD_F32", "SMEM_FLUSH_ADD_I32"):
                    cnt, var = desc(imm)
                    tgt = self._u(self.vars[var]).copy()
                    bins = smem[imm]
                    if name.endswith("F32"):             # a bin still holding -0.0 adds nothing and is skipped
                        tgt[:cnt] = np.where(bins != NEG_ZERO, self._u(f(tgt[:cnt]) + f(bins)), tgt[:cnt])
                    else: tgt[:cnt] = tgt[:cnt] + bins
                    self.vars[var] = tgt.view(self.vars[var].dtype)
                    return
                elif name == "GATHER_32_SMEM":
                    tab = smem[imm]; m = (B != 0) & (R < len(tab))
                    R = np.where(m, tab[np.where(m, R, 0)], np.uint32(0))
                elif name == "GATHER_32":
                    src = self._u(self.vars[gs_target(imm)]); m = (B != 0) & (R < len(src))
                    R = np.where(m, src[np.where(m, R, 0)], np.uint32(0))
                elif name in ("SCATTER_ADD_F32_SMEM", "SCATTER_ADD_I32_SMEM", "SCATTER_ADD_F32", "SCATTER_ADD_I32", "SCATTER_32"):
                    if name.endswith("_SMEM"):
                        tgt = smem[imm]
                    else:
                        var = gs_target(imm); tgt = self._u(self.vars[var]).copy()
                    m = (C != 0) & (R < len(tgt))
                    ii, vv = R[m], B[m]
                    if name == "SCATTER_32": tgt[ii] = vv
                    elif "F32" in name:
                        tf = tgt.view(np.float32)
                        for k_, v_ in zip(ii.tolist(), vv.view(np.float32).tolist()):      # element order, one rounding each
                            tf[k_] = np.float32(tf[k_] + np.float32(v_))
                    else: np.add.at(tgt, ii, vv)
                    if not name.endswith("_SMEM"):
                        self.vars[var] = tgt.view(self.vars[var].dtype)
                    return
                elif name == "RACC": state["R"] = R; racc(dst, imm); return
                elif name == "RFIN": rfin(B, Bh, imm, dst); return
                else:
                    raise Unsupported(name)
            state["R"] = np.ascontiguousarray(R).astype(np.uint32, copy=False)
            if flags & F_RACC:
                racc(dst, ca)
            if flags & F_STG:
                store_var(var_of_uniform(imm), state["R"])
            if flags & F_ST:
                slots[dst] = state["R"].copy()
                if flags & F_R64:
                    slots[dst + 1] = state["Rh"].copy()

        for ins in sw["init"]:
            execute(ins)
        for ins in sw["body"]:
            execute(ins)
        for ins in sw["fini"]:
            execute(ins)
