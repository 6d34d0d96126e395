"""Python mirror of enoki::DiffArray<CUDAArray<float>> (include/enoki/autodiff.h:126-1412).

`FloatD` carries a primal `Float32` and a tape node index; every differentiable op
computes the primal through the evaluator and registers the local partials of
SURVEY.md Appendix B as edge weights via the C ABI tape (ek_tape_*).  The heavy
lifting -- backward() -- runs in enoki_b200/csrc/ek_tape.cpp + ek_adjoint.cu.
"""
import ctypes
import numpy as np

from . import _lib

EK_FLOAT32 = 10


def _l():
    return _lib.load()


def _e():
    from . import EnokiError
    return EnokiError(_l().ek_last_error().decode())


class FloatD:
    """DiffArray<CUDAArray<float>>: {Type m_value; uint32 m_index} (autodiff.h:1410-1411)."""
    __slots__ = ("value", "index")

    def __init__(self, value=0.0, index=0):
        from . import Float32, CUDAArray
        if isinstance(value, FloatD):
            self.value, self.index = value.value, value.index
            _l().ek_tape_inc_ref_ext(EK_FLOAT32, self.index)
            return
        self.value = value if isinstance(value, CUDAArray) else Float32(value)
        self.index = index

    def __del__(self):
        try:
            if self.index:
                _l().ek_tape_dec_ref_ext(EK_FLOAT32, self.index)
        except Exception:
            pass

    # ---- tape plumbing
    @staticmethod
    def _node(label, value, inputs, weights):
        """Tape::append (autodiff.cpp:266-308): inputs = FloatD list, weights = Float32 list."""
        from . import Float32
        n = len(inputs)
        idx = (ctypes.c_uint32 * n)(*[i.index for i in inputs])
        if not any(idx):
            return FloatD(value, 0)
        ws = [w if hasattr(w, "index") else Float32(w) for w in weights]
        wh = (ctypes.c_uint32 * n)(*[w.index for w in ws])
        node = _l().ek_tape_append(EK_FLOAT32, label.encode(), value.size(), n, idx, wh)
        if node == 0:
            raise _e()
        return FloatD(value, node)

    def requires_gradient(self):
        return self.index != 0

    def set_requires_gradient(self, value=True):
        # autodiff.h:1270-1281
        if value and self.index == 0:
            self.index = _l().ek_tape_append_leaf(EK_FLOAT32, self.value.size())
        elif not value and self.index != 0:
            _l().ek_tape_dec_ref_ext(EK_FLOAT32, self.index)
            self.index = 0

    def size(self):
        return self.value.size()

    def numpy(self):
        return self.value.numpy()

    # ---- arithmetic with the partials of Appendix B
    @staticmethod
    def _c(x):
        return x if isinstance(x, FloatD) else FloatD(x)

    def __add__(self, o):
        o = FloatD._c(o)
        return FloatD._node("add", self.value + o.value, [self, o], [1.0, 1.0])

    __radd__ = __add__

    def __sub__(self, o):
        o = FloatD._c(o)
        return FloatD._node("sub", self.value - o.value, [self, o], [1.0, -1.0])

    def __rsub__(self, o):
        return FloatD._c(o) - self

    def __mul__(self, o):
        o = FloatD._c(o)
        return FloatD._node("mul", self.value * o.value, [self, o], [o.value, self.value])

    __rmul__ = __mul__

    def __truediv__(self, o):
        from . import rcp
        o = FloatD._c(o)
        rb = rcp(o.value)                                  # autodiff.h:258-272
        return FloatD._node("div", self.value / o.value, [self, o], [rb, -self.value * (rb * rb)])

    def __rtruediv__(self, o):
        return FloatD._c(o) / self

    def __neg__(self):
        return FloatD._node("neg", -self.value, [self], [-1.0])


def _unary(label, f, dfdx):
    def op(x):
        if not isinstance(x, FloatD):
            return f(x)
        r = f(x.value)
        if x.index == 0:
            return FloatD(r, 0)
        return FloatD._node(label, r, [x], [dfdx(x.value, r)])
    return op


def _build():
    from . import sin as _sin, cos as _cos, exp as _exp, log as _log, sqrt as _sqrt, rcp as _rcp, Float32, UInt32, reinterpret
    from . import tan as _tan, cot as _cot, asin as _asin, acos as _acos, atan as _atan, rsqrt as _rsqrt
    from . import sinh as _sinh, cosh as _cosh, tanh as _tanh, asinh as _asinh, acosh as _acosh, atanh as _atanh, cbrt as _cbrt
    from . import erf as _erf, erfc as _erfc, erfinv as _erfinv

    def _sign(a):
        # sign(a) = (sign_mask & a) | 1.0 (array_router.h:372): -1 at -0.0 and at NaNs with the sign bit set
        return reinterpret(Float32, (reinterpret(UInt32, a) & 0x80000000) | 0x3f800000)

    g = {}
    g["sin"] = _unary("sin", _sin, lambda a, r: _cos(a))
    g["cos"] = _unary("cos", _cos, lambda a, r: -_sin(a))
    g["exp"] = _unary("exp", _exp, lambda a, r: r)
    g["log"] = _unary("log", _log, lambda a, r: _rcp(a))
    g["sqrt"] = _unary("sqrt", _sqrt, lambda a, r: Float32(0.5) / r)       # autodiff.h:353-364
    g["rcp"] = _unary("rcp", _rcp, lambda a, r: -(r * r))                  # autodiff.h:379-390
    g["abs"] = _unary("abs", lambda a: abs(a), lambda a, r: _sign(a))      # autodiff.h:341-351

    def _sqr_sec(a):
        s = _rcp(_cos(a))
        return s * s

    def _neg_sqr_csc(a):
        c = _rcp(_sin(a))
        return -(c * c)

    g["tan"] = _unary("tan", _tan, lambda a, r: _sqr_sec(a))                    # autodiff.h:532-542: sqr(sec(a))
    g["cot"] = _unary("cot", _cot, lambda a, r: _neg_sqr_csc(a))                # autodiff.h:570-580: -sqr(csc(a))
    g["asin"] = _unary("asin", _asin, lambda a, r: _rsqrt(1.0 - a * a))         # autodiff.h:582-592
    g["acos"] = _unary("acos", _acos, lambda a, r: -_rsqrt(1.0 - a * a))        # autodiff.h:594-604
    g["atan"] = _unary("atan", _atan, lambda a, r: _rcp(1.0 + a * a))           # autodiff.h:606-616

    def _sqr_sech(a):
        s = _rcp(_cosh(a))
        return s * s

    g["sinh"] = _unary("sinh", _sinh, lambda a, r: _cosh(a))                    # autodiff.h:635-645
    g["cosh"] = _unary("cosh", _cosh, lambda a, r: _sinh(a))                    # autodiff.h:647-657
    g["tanh"] = _unary("tanh", _tanh, lambda a, r: _sqr_sech(a))                # autodiff.h:685-696: sqr(sech(a))
    g["asinh"] = _unary("asinh", _asinh, lambda a, r: _rsqrt(1.0 + a * a))      # autodiff.h:698-708
    g["acosh"] = _unary("acosh", _acosh, lambda a, r: _rsqrt(a * a - 1.0))      # autodiff.h:710-720
    g["atanh"] = _unary("atanh", _atanh, lambda a, r: _rcp(1.0 - a * a))        # autodiff.h:722-732
    g["cbrt"] = _unary("cbrt", _cbrt, lambda a, r: 1.0 / (3.0 * (r * r)))      # autodiff.h:366-377

    # autodiff.h has no weights for special.h's functions: these are the analytic derivatives
    two_over_sqrt_pi, sqrt_pi_over_2 = 1.1283791670955126, 0.886226925452758
    g["erf"] = _unary("erf", _erf, lambda a, r: two_over_sqrt_pi * _exp(-(a * a)))
    g["erfc"] = _unary("erfc", _erfc, lambda a, r: -two_over_sqrt_pi * _exp(-(a * a)))
    g["erfinv"] = _unary("erfinv", _erfinv, lambda a, r: sqrt_pi_over_2 * _exp(r * r))
    return g


_ops = None


def _op(name):
    global _ops
    if _ops is None:
        _ops = _build()
    return _ops[name]


def sin(x): return _op("sin")(x)
def cos(x): return _op("cos")(x)
def exp(x): return _op("exp")(x)
def log(x): return _op("log")(x)
def sqrt(x): return _op("sqrt")(x)
def rcp(x): return _op("rcp")(x)
def abs_(x): return _op("abs")(x)
def tan(x): return _op("tan")(x)
def cot(x): return _op("cot")(x)
def asin(x): return _op("asin")(x)
def acos(x): return _op("acos")(x)
def atan(x): return _op("atan")(x)
def sinh(x): return _op("sinh")(x)
def cosh(x): return _op("cosh")(x)
def tanh(x): return _op("tanh")(x)
def asinh(x): return _op("asinh")(x)
def acosh(x): return _op("acosh")(x)
def atanh(x): return _op("atanh")(x)
def cbrt(x): return _op("cbrt")(x)


def erf(x):
    """erf(x); weight (2 / sqrt(pi)) * exp(-x * x)"""
    return _op("erf")(x)


def erfc(x):
    """erfc(x); weight -(2 / sqrt(pi)) * exp(-x * x)"""
    return _op("erfc")(x)


def erfinv(x):
    """erfinv(x); weight (sqrt(pi) / 2) * exp(r * r), where r = erfinv(x)"""
    return _op("erfinv")(x)


def atan2(y, x):
    """autodiff.h:618-633: il2 = rcp(sqr(y) + sqr(x)), weights (il2 * x, -il2 * y)."""
    from . import atan2 as _atan2, rcp as _rcp
    y, x = FloatD._c(y), FloatD._c(x)
    r = _atan2(y.value, x.value)
    if y.index == 0 and x.index == 0:
        return FloatD(r, 0)
    il2 = _rcp(y.value * y.value + x.value * x.value)
    return FloatD._node("atan2", r, [y, x], [il2 * x.value, -il2 * y.value])


def fmadd(a, b, c):
    """autodiff.h:274-286: weights (b, a, 1)."""
    from . import fmadd as _fmadd
    a, b, c = FloatD._c(a), FloatD._c(b), FloatD._c(c)
    return FloatD._node("fmadd", _fmadd(a.value, b.value, c.value), [a, b, c], [b.value, a.value, 1.0])


def hsum(x):
    """autodiff.h:1052-1062: size-1 target, weight 1."""
    from . import hsum as _hsum
    r = _hsum(x.value)
    if x.index == 0:
        return FloatD(r, 0)
    from . import Float32
    one = Float32(1.0)
    idx = (ctypes.c_uint32 * 1)(x.index)
    wh = (ctypes.c_uint32 * 1)(one.index)
    node = _l().ek_tape_append(EK_FLOAT32, b"hsum", 1, 1, idx, wh)
    return FloatD(r, node)


def detach(x):
    return x.value


def set_requires_gradient(x, value=True):
    x.set_requires_gradient(value)


def gradient(x):
    """autodiff.h:1300-1304 / autodiff.cpp:796-802"""
    from . import Float32
    h = _l().ek_tape_gradient(EK_FLOAT32, x.index)
    if h == 0:
        msg = _l().ek_last_error().decode()
        if msg:
            raise _e()
        return Float32.zero(x.size())
    _l().ek_inc_ref_ext(h)
    return Float32.from_index(h)


def backward(x, free_graph=True):
    """autodiff.h:1490-1492 -> Tape::backward (autodiff.cpp:804-811,838-910)"""
    if _l().ek_tape_backward(EK_FLOAT32, x.index, int(free_graph)) != 0:
        raise _e()


def set_gradient(x, value, backward=True):
    """autodiff.h:1306-1312 / autodiff.cpp:822-836: seeds the gradient of `x` (a Float32 array) and schedules the
    nodes reachable from it; follow with backward_static() (FloatD.backward() of the reference's Python module)."""
    from . import Float32, CUDAArray
    v = value if isinstance(value, CUDAArray) else Float32(value)
    if _l().ek_tape_set_gradient(EK_FLOAT32, x.index, v.index, int(backward)) != 0:
        raise _e()


def backward_static(free_graph=True):
    """src/python/cuda_autodiff_1d.cpp:23-35 `FloatD.backward()`"""
    if _l().ek_tape_backward_static(EK_FLOAT32, int(free_graph)) != 0:
        raise _e()


def forward(x, free_graph=True):
    if _l().ek_tape_forward(EK_FLOAT32, x.index, int(free_graph)) != 0:
        raise _e()
