"""enoki_b200 -- H100-native backend for Enoki's CUDAArray evaluator and DiffArray tape.

Python host-side mirror of the reference's `enoki.cuda` / `enoki.cuda_autodiff`
modules (src/python/cuda*.cpp): thin array classes that record operations through
the C ABI in include/enoki_b200.h.  Nothing is computed in Python and there is no
CPU fallback: every value is produced by the sm_90a kernels behind `cuda_eval()`.

    from enoki_b200 import Float32, UInt32, sin, exp, fmadd, hsum, cuda_eval
    a = Float32.copy(np_array); b = fmadd(a, a, 1.0); print(hsum(sin(b)).numpy())
"""
import ctypes
import numpy as np

from . import _lib
from ._lib import ek_stats

# ---- enums (include/enoki_b200.h) -------------------------------------------------
(EK_INVALID, EK_INT8, EK_UINT8, EK_INT16, EK_UINT16, EK_INT32, EK_UINT32, EK_INT64,
 EK_UINT64, EK_FLOAT16, EK_FLOAT32, EK_FLOAT64, EK_BOOL, EK_POINTER) = range(14)

_OPS = ["INVALID", "LITERAL", "INDEX", "MOV", "CVT", "BITCAST", "NEG", "ABS", "SQRT", "RCP", "RSQRT",
        "EXP", "LOG", "SIN", "COS", "FLOOR", "CEIL", "ROUND", "TRUNC", "FLOOR2INT", "CEIL2INT", "NOT",
        "POPC", "CLZ", "CTZ", "ADD", "SUB", "MUL", "MULHI", "DIV", "MOD", "MIN", "MAX", "SHL", "SHR",
        "AND", "OR", "XOR", "GT", "GE", "LT", "LE", "EQ", "NE", "MUL_NZ", "FMA", "SELECT", "FMA_NZ",
        "GATHER", "SCATTER", "SCATTER_ADD", "HSUM", "HPROD", "HMAX", "HMIN", "ALL", "ANY", "COUNT", "PRINTF",
        "TAN", "COT", "ASIN", "ACOS", "ATAN", "ATAN2", "SINH", "COSH", "TANH", "ASINH", "ACOSH", "ATANH", "CBRT"]
# special.h's functions, numbered after EK_OP_CBRT (include/enoki_b200.h) in a group of their own, like their sweep
# operations (EK_FX_SPEC)
_OPS_SPECIAL = ["ERF", "ERFC", "ERFINV", "LGAMMA", "TGAMMA"]
OP = {n: i for i, n in enumerate(_OPS + _OPS_SPECIAL)}
# the remaining Float32 functions of array_math.h and special.h, numbered after EK_OP_TGAMMA (their sweep operations:
# EK_FX_MATH); a table of their own, so that OP keeps the opcodes it held before they existed
_OPS_MATH = ["POW", "FREXP_M", "FREXP_E", "HYPOT", "DAWSON", "ERFI"]
OP_MATH = {n: len(OP) + i for i, n in enumerate(_OPS_MATH)}
# special.h's Carlson integrals, numbered after EK_OP_ERFI (their sweep operations: EK_FX_ELL), in a table of their own
_OPS_ELL = ["CARLSON_RF", "CARLSON_RD", "CARLSON_RC"]
OP_ELL = {n: len(OP) + len(OP_MATH) + i for i, n in enumerate(_OPS_ELL)}
_OPCODE = {**OP, **OP_MATH, **OP_ELL}

_NP = {EK_INT8: np.int8, EK_UINT8: np.uint8, EK_INT16: np.int16, EK_UINT16: np.uint16,
       EK_INT32: np.int32, EK_UINT32: np.uint32, EK_INT64: np.int64, EK_UINT64: np.uint64,
       EK_FLOAT16: np.float16, EK_FLOAT32: np.float32, EK_FLOAT64: np.float64, EK_BOOL: np.bool_}


class EnokiError(RuntimeError):
    """Raised where the reference throws std::runtime_error (jit.cu:207-212,366-371,722-725,777-782)."""


def lib():
    return _lib.load()


def _check(handle_or_rc, ok):
    if not ok:
        raise EnokiError(lib().ek_last_error().decode())
    return handle_or_rc


def _append(t, op, a=0, b=0, c=0, imm=0):
    h = lib().ek_trace_append(t, _OPCODE[op], a, b, c, imm)
    return _check(h, h != 0)


# ---- array classes -------------------------------------------------------------------
class CUDAArray:
    """Mirror of enoki::CUDAArray<T> (include/enoki/cuda.h:205-954): a ref-counted trace handle."""
    Type = EK_INVALID
    __slots__ = ("index",)

    def __init__(self, value=None):
        self.index = 0
        if value is None:
            return
        if isinstance(value, CUDAArray):
            if value.Type == self.Type:
                self.index = value.index
                lib().ek_inc_ref_ext(self.index)
            else:                                  # converting constructor, cuda.h:236-247
                self.index = _append(self.Type, "CVT", value.index)
        elif isinstance(value, (np.ndarray, list, tuple)):
            arr = np.ascontiguousarray(value, dtype=_NP[self.Type])
            h = lib().ek_var_copy_to_device(self.Type, arr.size, arr.ctypes.data)
            self.index = _check(h, h != 0)
        else:                                      # scalar literal, cuda.h:267-317
            # (a Float16 literal is half(float(value)), the reference's converting constructor: two roundings)
            val = np.array([value], dtype=np.float32 if self.Type == EK_FLOAT16 else _NP[self.Type]).astype(_NP[self.Type])
            bits = val.view(
                {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[np.dtype(_NP[self.Type]).itemsize])[0]
            self.index = _append(self.Type, "LITERAL", imm=int(bits))

    def __del__(self):
        try:
            if self.index:
                lib().ek_dec_ref_ext(self.index)
        except Exception:
            pass

    # -- construction helpers (cuda.h:641-691, 796-802)
    @classmethod
    def from_index(cls, index):
        r = cls.__new__(cls)
        r.index = index
        return r

    @classmethod
    def copy(cls, array):
        return cls(np.asarray(array))

    @classmethod
    def map(cls, ptr, size, dealloc=False):
        h = lib().ek_var_register(cls.Type, size, ptr, int(dealloc))
        return cls.from_index(_check(h, h != 0))

    @classmethod
    def empty(cls, size):
        p = lib().ek_malloc(size * np.dtype(_NP[cls.Type]).itemsize)
        return cls.map(p, size, True)

    @classmethod
    def zero(cls, size=1):
        if size == 1:
            return cls(0)
        es = np.dtype(_NP[cls.Type]).itemsize
        p = lib().ek_malloc(size * es)
        lib().ek_fill(p, 1, 0, size * es)
        return cls.map(p, size, True)

    @classmethod
    def full(cls, value, size=1):
        r = cls(value)
        if size != 1:
            r.index = _check(*(lambda h: (h, h != 0))(lib().ek_var_set_size(r.index, size, 1)))
        return r

    @classmethod
    def arange(cls, size):
        idx = UInt32.from_index(_append(EK_UINT32, "INDEX"))
        h = lib().ek_var_set_size(idx.index, size, 0)
        _check(h, h != 0)
        return idx if cls is UInt32 else cls(idx)

    @classmethod
    def linspace(cls, lo, hi, size):
        idx = UInt32.arange(size)
        step = (np.float32(hi) - np.float32(lo)) / np.float32(size - 1) if cls.Type == EK_FLOAT32 \
            else (hi - lo) / (size - 1)
        return fmadd(cls(idx), cls(step), cls(lo))

    # -- queries
    def size(self):
        return lib().ek_var_size(self.index) if self.index else 0

    def __len__(self):
        return self.size()

    def data(self):
        self.eval()
        return lib().ek_var_ptr(self.index)

    def eval(self):
        _check(0, lib().ek_eval_var(self.index) == 0)
        return self

    def numpy(self):
        """Evaluate and copy to host (src/python/common.h:1085-1110 semantics)."""
        n = self.size()
        self.eval()
        lib().ek_sync()
        out = np.empty(n, dtype=_NP[self.Type])
        ptr = lib().ek_var_ptr(self.index)
        if ptr is None:
            raise EnokiError("numpy(): variable has no storage")
        lib().ek_memcpy_from_device(out.ctypes.data, ptr, out.nbytes)
        return out

    def coeff(self, i):
        out = np.zeros(1, dtype=_NP[self.Type])
        _check(0, lib().ek_fetch_element(out.ctypes.data, self.index, i, out.itemsize) == 0)
        return out[0]

    def set_label(self, label):
        lib().ek_var_set_label(self.index, label.encode())
        return self

    # -- helpers
    def _coerce(self, other):
        return other if isinstance(other, CUDAArray) else type(self)(other)

    def _bin(self, op, other, rtype=None, swap=False):
        o = self._coerce(other)
        a, b = (o, self) if swap else (self, o)
        cls = rtype or type(self)
        return cls.from_index(_append(cls.Type, op, a.index, b.index))

    def _un(self, op, rtype=None):
        cls = rtype or type(self)
        return cls.from_index(_append(cls.Type, op, self.index))

    # -- arithmetic (cuda.h:341-427)
    def __add__(self, o): return self._bin("ADD", o)
    def __radd__(self, o): return self._bin("ADD", o, swap=True)
    def __sub__(self, o): return self._bin("SUB", o)
    def __rsub__(self, o): return self._bin("SUB", o, swap=True)
    def __mul__(self, o): return self._bin("MUL", o)
    def __rmul__(self, o): return self._bin("MUL", o, swap=True)
    def __truediv__(self, o): return self._bin("DIV", o)
    def __rtruediv__(self, o): return self._bin("DIV", o, swap=True)
    def __floordiv__(self, o): return self._bin("DIV", o)
    def __mod__(self, o): return self._bin("MOD", o)
    def __neg__(self): return self._un("NEG")
    def __abs__(self): return self._un("ABS")
    def __invert__(self): return self._un("NOT")
    def __and__(self, o): return self._bin("AND", o)
    def __or__(self, o): return self._bin("OR", o)
    def __xor__(self, o): return self._bin("XOR", o)
    def __lshift__(self, o): return self._bin("SHL", o)
    def __rshift__(self, o): return self._bin("SHR", o)
    def __gt__(self, o): return self._bin("GT", o, Mask)
    def __ge__(self, o): return self._bin("GE", o, Mask)
    def __lt__(self, o): return self._bin("LT", o, Mask)
    def __le__(self, o): return self._bin("LE", o, Mask)
    def eq_(self, o): return self._bin("EQ", o, Mask)
    def neq_(self, o): return self._bin("NE", o, Mask)


def _make(name, t):
    return type(name, (CUDAArray,), {"Type": t, "__slots__": ()})


Float16 = _make("Float16", EK_FLOAT16)     # storage only: convert to Float32 to compute (DESIGN.md 4)
Float32 = _make("Float32", EK_FLOAT32)
Float64 = _make("Float64", EK_FLOAT64)
Int8 = _make("Int8", EK_INT8)
UInt8 = _make("UInt8", EK_UINT8)
Int16 = _make("Int16", EK_INT16)
UInt16 = _make("UInt16", EK_UINT16)
Int32 = _make("Int32", EK_INT32)
UInt32 = _make("UInt32", EK_UINT32)
Int64 = _make("Int64", EK_INT64)
UInt64 = _make("UInt64", EK_UINT64)
Mask = _make("Mask", EK_BOOL)

_BY_TYPE = {c.Type: c for c in (Float16, Float32, Float64, Int8, UInt8, Int16, UInt16, Int32, UInt32, Int64, UInt64, Mask)}


# ---- free functions (array_router.h / array_math.h names) -------------------------------
def _unary(op):
    def f(x):
        return x._un(op)
    f.__name__ = op.lower()
    return f


sqrt, rcp, rsqrt, exp, log, sin, cos = (_unary(o) for o in ("SQRT", "RCP", "RSQRT", "EXP", "LOG", "SIN", "COS"))
floor, ceil, round_, trunc = (_unary(o) for o in ("FLOOR", "CEIL", "ROUND", "TRUNC"))
popcnt, lzcnt, tzcnt = (_unary(o) for o in ("POPC", "CLZ", "CTZ"))
abs_ = _unary("ABS")
# Float32 only: one node each, bit for bit the single precision branch of array_math.h (DESIGN.md 4)
tan, cot, asin, acos, atan = (_unary(o) for o in ("TAN", "COT", "ASIN", "ACOS", "ATAN"))
sinh, cosh, tanh, asinh, acosh, atanh, cbrt = (_unary(o) for o in ("SINH", "COSH", "TANH", "ASINH", "ACOSH", "ATANH", "CBRT"))
# Float32 only: one node each, bit for bit the single precision branch of special.h (DESIGN.md 4)
erf, erfc, erfinv, lgamma, tgamma = (_unary(o) for o in ("ERF", "ERFC", "ERFINV", "LGAMMA", "TGAMMA"))


def sincosh(x):
    """(sinh(x), cosh(x)): array_math.h:1067-1127 records the same operations as the two functions"""
    return sinh(x), cosh(x)


def atan2(y, x):
    """atan2(y, x) (array_math.h:603-664); either operand may be a Python number"""
    cls = next(type(v) for v in (y, x) if isinstance(v, CUDAArray))
    y, x = (v if isinstance(v, CUDAArray) else cls(v) for v in (y, x))
    return y._bin("ATAN2", x)


# Float32 only: one node each, bit for bit the single precision bodies of array_math.h and special.h (DESIGN.md 4)
dawson, erfi = (_unary(o) for o in ("DAWSON", "ERFI"))


def _binary(op, doc):
    def f(x, y):
        cls = next(type(v) for v in (x, y) if isinstance(v, CUDAArray))
        x, y = (v if isinstance(v, CUDAArray) else cls(v) for v in (x, y))
        return x._bin(op, y)
    f.__name__, f.__doc__ = op.lower(), doc
    return f


pow_ = _binary("POW", "pow(x, y) = exp(log(x) * y) (array_math.h:956-958); either operand may be a Python number")
hypot = _binary("HYPOT", "hypot(a, b) (array_math.h:1362-1379); either operand may be a Python number")


def frexp(x):
    """(mantissa, exponent) of array_math.h:682-709, both Float32"""
    return x._un("FREXP_M"), x._un("FREXP_E")


def _operands(*args):
    """the arguments as arrays of the first array argument's type (Float32 when all are Python numbers)"""
    cls = next((type(v) for v in args if isinstance(v, CUDAArray)), Float32)
    return [v if isinstance(v, CUDAArray) else cls(v) for v in args]


# Float32 only: one node each, bit for bit the single precision bodies of special.h, their duplication loops run per
# element on the device (DESIGN.md 4); any argument may be a Python number.  No autodiff: the reference has no
# derivatives for them.
def carlson_rf(x, y, z):
    """R_F(x, y, z) (special.h:325-366)"""
    x, y, z = _operands(x, y, z)
    return type(x).from_index(_append(x.Type, "CARLSON_RF", x.index, y.index, z.index))


def carlson_rd(x, y, z):
    """R_D(x, y, z) (special.h:379-432)"""
    x, y, z = _operands(x, y, z)
    return type(x).from_index(_append(x.Type, "CARLSON_RD", x.index, y.index, z.index))


def carlson_rc(x, y):
    """R_C(x, y) (special.h:445-482)"""
    x, y = _operands(x, y)
    return x._bin("CARLSON_RC", y)


def comp_ellint_1(k):
    """K(k) = carlson_rf(0, 1 - k^2, 1) (special.h:566-572): k is squared, unlike Mathematica's EllipticK"""
    return carlson_rf(0.0, 1.0 - k * k, 1.0)


def comp_ellint_2(k):
    """E(k) = carlson_rf(xyz) - 1/3 k^2 carlson_rd(xyz), xyz = (0, 1 - k^2, 1) (special.h:599-606)"""
    k2 = k * k
    y = 1.0 - k2
    return carlson_rf(0.0, y, 1.0) - (1.0 / 3.0) * k2 * carlson_rd(0.0, y, 1.0)


def sincos(x):
    return sin(x), cos(x)


def fmadd(a, b, c):
    cls = next(type(v) for v in (a, b, c) if isinstance(v, CUDAArray))
    a, b, c = (v if isinstance(v, CUDAArray) else cls(v) for v in (a, b, c))
    return cls.from_index(_append(cls.Type, "FMA", a.index, b.index, c.index))


def fmsub(a, b, c): return fmadd(a, b, -c)
def fnmadd(a, b, c): return fmadd(-a, b, c)
def fnmsub(a, b, c): return -fmadd(a, b, c)
def min_(a, b): return a._bin("MIN", b)
def max_(a, b): return a._bin("MAX", b)
def mulhi(a, b): return a._bin("MULHI", b)
def eq(a, b): return a.eq_(b)
def neq(a, b): return a.neq_(b)
def sqr(a): return a * a
def mul_nz(a, b): return a._bin("MUL_NZ", b)


def fma_nz(a, b, c):
    return type(a).from_index(_append(a.Type, "FMA_NZ", a.index, b.index, c.index))


def select(m, t, f):
    cls = next(type(v) for v in (t, f) if isinstance(v, CUDAArray))
    t, f = (v if isinstance(v, CUDAArray) else cls(v) for v in (t, f))
    return cls.from_index(_append(cls.Type, "SELECT", m.index, t.index, f.index))


def reinterpret(cls, x):
    return cls.from_index(_append(cls.Type, "BITCAST", x.index))


def floor2int(cls, x): return cls.from_index(_append(cls.Type, "FLOOR2INT", x.index))
def ceil2int(cls, x): return cls.from_index(_append(cls.Type, "CEIL2INT", x.index))


def _reduce(op, x, rtype=None):
    cls = rtype or type(x)
    if x.size() == 1 and op in ("HSUM", "HPROD", "HMAX", "HMIN"):
        return x                                  # cuda.h:693-697
    return cls.from_index(_append(cls.Type, op, x.index))


def hsum(x): return _reduce("HSUM", x)
def hprod(x): return _reduce("HPROD", x)
def hmax(x): return _reduce("HMAX", x)
def hmin(x): return _reduce("HMIN", x)
def all_(m): return bool(_reduce("ALL", m, Mask).coeff(0))
def any_(m): return bool(_reduce("ANY", m, Mask).coeff(0))
def count(m): return int(_reduce("COUNT", m, UInt32).coeff(0))


def gather(cls, source, index, mask=True):
    """gather<cls>(source_array, index, mask): include/enoki/array_struct.h:8-41 + cuda.h:845-864."""
    mask = mask if isinstance(mask, CUDAArray) else Mask(mask)
    _check(0, lib().ek_set_scatter_gather_operand(source.index, 1) == 0)
    try:
        ptr = lib().ek_var_register_ptr(lib().ek_var_ptr(source.index))
        try:
            stride = np.dtype(_NP[cls.Type]).itemsize
            r = cls.from_index(_append(cls.Type, "GATHER", ptr, index.index, mask.index, stride))
        finally:
            lib().ek_dec_ref_ext(ptr)
    finally:
        lib().ek_set_scatter_gather_operand(0, 0)
    return r


def _scatter(op, target, value, index, mask):
    mask = mask if isinstance(mask, CUDAArray) else Mask(mask)
    value = value if isinstance(value, CUDAArray) else type(target)(value)
    _check(0, lib().ek_set_scatter_gather_operand(target.index, 0) == 0)
    try:
        ptr = lib().ek_var_register_ptr(lib().ek_var_ptr(target.index))
        try:
            stride = np.dtype(_NP[value.Type]).itemsize
            h = _append(value.Type if op == "SCATTER_ADD" else EK_UINT64, op, ptr, index.index, mask.index,
                        (stride << 32) | value.index)
            lib().ek_var_mark_side_effect(h)
        finally:
            lib().ek_dec_ref_ext(ptr)
        lib().ek_var_mark_dirty(target.index)          # array_struct.h:85,119
    finally:
        lib().ek_set_scatter_gather_operand(0, 0)


def scatter(target, value, index, mask=True):
    """include/enoki/array_struct.h:56-89 + cuda.h:866-890"""
    _scatter("SCATTER", target, value, index, mask)


def scatter_add(target, value, index, mask=True):
    """include/enoki/array_struct.h:91-123 + cuda.h:892-905"""
    _scatter("SCATTER_ADD", target, value, index, mask)


def partition(ptrs):
    """Virtual-call dispatch grouping of a UInt64 pointer array (CUDAArray<T *>::partition_(), cuda.h:814-843):
    [(pointer, UInt32 indices holding it)], pointers ascending, indices ascending inside a group."""
    if ptrs.Type != EK_UINT64:
        raise TypeError("partition(): expects a UInt64 array")
    ptrs.eval()
    L = lib()
    uniq, counts, lists = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    _check(0, L.ek_partition(ptrs.size(), ptrs.data(), ctypes.byref(uniq), ctypes.byref(counts),
                             ctypes.byref(lists)) == 0)
    try:
        k = ctypes.cast(counts, ctypes.POINTER(ctypes.c_uint32))[0]
        sizes = np.ctypeslib.as_array(ctypes.cast(counts, ctypes.POINTER(ctypes.c_uint32)), shape=(k + 1,))[1:].copy()
        keys = np.ctypeslib.as_array(ctypes.cast(uniq, ctypes.POINTER(ctypes.c_uint64)), shape=(k,)).copy()
        ptrs_d = np.ctypeslib.as_array(ctypes.cast(lists, ctypes.POINTER(ctypes.c_uint64)), shape=(k,)).copy()
    finally:
        L.ek_host_free(uniq)
        L.ek_host_free(counts)
    try:
        groups = []
        for g in range(k):                 # each list is owned by its UInt32 from here on (dealloc = true)
            groups.append((int(keys[g]), UInt32.map(int(ptrs_d[g]), int(sizes[g]), True)))
            ptrs_d[g] = 0
    finally:
        for p in ptrs_d[ptrs_d != 0]:
            L.ek_free(ctypes.c_void_p(int(p)))
        libc = ctypes.CDLL(None)
        libc.free.argtypes = [ctypes.c_void_p]
        libc.free(lists)
    return groups


def cuda_printf(fmt, *args):
    """enoki::cuda_printf (array_router.h:971-975): record a print of up to 3 arrays.  The evaluation that runs it
    writes one line per element to C stdout, in recording order, with the values the arrays had when the print was
    recorded.  The format is checked now (see ek_printf.cpp); a rejected one raises EnokiError and records nothing.
    Print a DiffArray through detach(x)."""
    for a in args:
        if not isinstance(a, CUDAArray):
            raise TypeError(f"cuda_printf(): arguments must be CUDA arrays, not {type(a).__name__}")
    idx = (ctypes.c_uint32 * max(len(args), 1))(*[a.index for a in args])
    _check(0, lib().ek_trace_printf(fmt.encode() if isinstance(fmt, str) else fmt, len(args), idx) == 0)


def cuda_eval():
    _check(0, lib().ek_eval() == 0)


def cuda_sync():
    lib().ek_sync()


def cuda_malloc_trim():
    lib().ek_malloc_trim()


def cuda_set_log_level(level):
    lib().ek_set_log_level(level)


def cuda_whos():
    return _lib.take_string(lib().ek_whos())


def debug_plan():
    """Textual listing of the sweep programs cuda_eval() would launch (host-only)."""
    p = lib().ek_debug_plan()
    if not p:
        raise EnokiError(lib().ek_last_error().decode())
    return _lib.take_string(p)


def debug_program():
    """The same as JSON with the complete sweep programs (consumed by tests/ek_emulator.py)."""
    import json
    p = lib().ek_debug_program()
    if not p:
        raise EnokiError(lib().ek_last_error().decode())
    return json.loads(_lib.take_string(p))


def stats():
    s = ek_stats()
    lib().ek_stats_get(ctypes.byref(s))
    return s


def device_count():
    return lib().ek_device_count()


from .autodiff import FloatD, backward, forward, gradient, set_requires_gradient, detach  # noqa: E402,F401
from .dlpack import from_dlpack  # noqa: E402,F401  (also installs __dlpack__ / __dlpack_device__ / from_dlpack)
