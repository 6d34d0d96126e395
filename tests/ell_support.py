"""TEST INFRASTRUCTURE for carlson_rf, carlson_rd and carlson_rc (EK_OP_CARLSON_RF ... EK_OP_CARLSON_RC): the plain-C
restatements of tests/ell_oracle.c, compiled into a temporary directory, and the numpy interpreter of
tests/ek_emulator.py taught the new sweep operations through them (together with the sets of tests/math_support.py)."""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

import math_support as ms
from ek_emulator import Emulator
from fast_kernel_emu import FastKernelEmulator

HERE = os.path.dirname(os.path.abspath(__file__))
TERNARY = ("carlson_rf", "carlson_rd")
BINARY = ("carlson_rc",)
ELL_DOPS = ("CARLSON_RF_F32", "CARLSON_RD_F32", "CARLSON_RC_F32", "CARLSON_RCR_F32")
_lib = None


def lib():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="ell_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libell_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=gnu11", "-ffp-contract=off", "-fno-math-errno",
                               "-mfma", "-fPIC", "-shared", os.path.join(HERE, "ell_oracle.c"), "-o", so, "-lm"])
        _lib = ctypes.CDLL(so)
    return _lib


def _P(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _f32(*args):
    args = np.broadcast_arrays(*(np.asarray(a, np.float32) for a in args))
    return [np.ascontiguousarray(a.ravel()) for a in args]


def call(name, *args):
    """carlson_rf / carlson_rd (x, y, z) or carlson_rc (x, y) of float32 arrays (broadcast), as the restatement computes
    them"""
    if name in TERNARY:
        x, y, z = _f32(*args)
        out = np.empty_like(x)
        lib().el_ternary_f32(TERNARY.index(name), _P(x), _P(y), _P(z), _P(out), ctypes.c_size_t(len(x)))
        return out
    x, y = _f32(*args)
    out = np.empty_like(x)
    lib().el_binary_f32(_P(x), _P(y), _P(out), ctypes.c_size_t(len(x)))
    return out


same_bits = ms.same_bits


def _ell(name, R, B, C):
    """the new sweep operations on the accumulator bits R and operand bits B, C; None for other names"""
    f = lambda v: np.ascontiguousarray(v).view(np.float32)
    if name == "CARLSON_RF_F32":
        return call("carlson_rf", f(R), f(B), f(C)).view(np.uint32)
    if name == "CARLSON_RD_F32":
        return call("carlson_rd", f(R), f(B), f(C)).view(np.uint32)
    if name == "CARLSON_RC_F32":
        return call("carlson_rc", f(R), f(B)).view(np.uint32)
    if name == "CARLSON_RCR_F32":
        return call("carlson_rc", f(B), f(R)).view(np.uint32)
    return None


class _EllMixin:
    """Routes the new operations through the restatements, the way math_support._MathMixin does: renamed with a CVT_
    prefix, they reach _exec64 first."""
    def run(self, program):
        ren = lambda n: "CVT_" + n if n in ELL_DOPS else n
        program = dict(program, ops=[ren(n) for n in program["ops"]], fops=[ren(n) for n in program["fops"]])
        return super().run(program)

    def _exec64(self, name, imm, R, Rh, B, Bh, C, Ch, staged, cb):
        r = _ell(name[4:], R, B, C) if name.startswith("CVT_") and name[4:] in ELL_DOPS else None
        return (r, Rh) if r is not None else super()._exec64(name, imm, R, Rh, B, Bh, C, Ch, staged, cb)


class EllEmulator(_EllMixin, ms._MathMixin, ms.ss._SpecMixin, ms.hs._HypMixin, ms.ts._TrigMixin, Emulator):
    pass


class EllKernelEmulator(_EllMixin, ms._MathMixin, ms.ss._SpecMixin, ms.hs._HypMixin, ms.ts._TrigMixin, FastKernelEmulator):
    """fast sweeps on the host-compiled kernel, the others on the interpreter"""
    pass
