"""TEST INFRASTRUCTURE for pow, frexp, hypot, dawson and erfi (EK_OP_POW ... EK_OP_ERFI): the plain-C
restatements of tests/math_oracle.c, compiled into a temporary directory, and the numpy interpreter of
tests/ek_emulator.py taught the new sweep operations through them (together with the special functions of
tests/special_support.py, the hyperbolic ones of tests/hyp_support.py and the trigonometric ones of
tests/trig_support.py)."""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

import hyp_support as hs
import special_support as ss
import trig_support as ts
from ek_emulator import Emulator
from fast_kernel_emu import FastKernelEmulator

HERE = os.path.dirname(os.path.abspath(__file__))
BINARY = ("pow", "hypot")
UNARY = ("frexp_m", "frexp_e", "dawson", "erfi")
MATH_DOPS = tuple(n.upper() + "_F32" for n in BINARY + UNARY) + tuple(n.upper() + "R_F32" for n in BINARY)
_lib = None


def lib():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="math_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libmath_oracle.so")
        oracle = os.path.join(os.path.dirname(HERE), "oracle")            # exp / log: liboracle.so's or_*
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=gnu11", "-D_GNU_SOURCE", "-ffp-contract=off",
                               "-fno-math-errno", "-fPIC", "-shared", os.path.join(HERE, "math_oracle.c"), "-o", so,
                               "-L" + oracle, "-loracle", "-Wl,-rpath," + oracle, "-lm"])
        _lib = ctypes.CDLL(so)
    return _lib


def _P(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def binary(name, x, y):
    """pow / hypot of the float32 arrays x and y (broadcast), as the restatement computes them"""
    x, y = np.broadcast_arrays(np.asarray(x, np.float32), np.asarray(y, np.float32))
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y); out = np.empty_like(x)
    lib().mt_binary_f32(BINARY.index(name), _P(x), _P(y), _P(out), ctypes.c_size_t(len(x)))
    return out


def unary(name, x):
    """frexp_m / frexp_e / dawson / erfi of the float32 array x, as the restatement computes them"""
    x = np.ascontiguousarray(x, np.float32); out = np.empty_like(x)
    lib().mt_unary_f32(UNARY.index(name), _P(x), _P(out), ctypes.c_size_t(len(x)))
    return out


def call(name, *args):
    return binary(name, *args) if name in BINARY else unary(name, *args)


same_bits = ts.same_bits


def _math(name, R, B):
    """the new sweep operations on the accumulator bits R (and operand bits B); None for other names"""
    f = lambda v: np.ascontiguousarray(v).view(np.float32)
    base = name[:-4].lower()
    if base in UNARY:
        return unary(base, f(R)).view(np.uint32)
    if base in BINARY:
        return binary(base, f(R), f(B)).view(np.uint32)
    if base.endswith("r") and base[:-1] in BINARY:
        return binary(base[:-1], f(B), f(R)).view(np.uint32)
    return None


class _MathMixin:
    """Routes the new operations through the restatements, the way trig_support._TrigMixin routes atan2: renamed with a
    CVT_ prefix (their uniform twins too), they reach _exec64 first."""
    def run(self, program):
        # (the fast kernel names the uniform twins X_UB; the interpreter decodes any X_U as X with a uniform B)
        ren = lambda n: "CVT_" + n if n in MATH_DOPS else "CVT_" + n[:-1] if n.endswith("_UB") and n[:-3] in MATH_DOPS else n
        program = dict(program, ops=[ren(n) for n in program["ops"]], fops=[ren(n) for n in program["fops"]])
        return super().run(program)

    def _exec64(self, name, imm, R, Rh, B, Bh, C, Ch, staged, cb):
        r = _math(name[4:], R, B) if name.startswith("CVT_") and name[4:] in MATH_DOPS else None
        return (r, Rh) if r is not None else super()._exec64(name, imm, R, Rh, B, Bh, C, Ch, staged, cb)


class MathEmulator(_MathMixin, ss._SpecMixin, hs._HypMixin, ts._TrigMixin, Emulator):
    pass


class MathKernelEmulator(_MathMixin, ss._SpecMixin, hs._HypMixin, ts._TrigMixin, FastKernelEmulator):
    """fast sweeps on the host-compiled kernel, the others on the interpreter"""
    pass
