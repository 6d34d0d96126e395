"""TEST INFRASTRUCTURE for the trigonometric operations (EK_OP_TAN ... EK_OP_ATAN2): the plain-C restatements of
tests/trig_oracle.c, compiled into a temporary directory, and the numpy interpreter of tests/ek_emulator.py taught the
seven new sweep operations through them."""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

from ek_emulator import Emulator
from fast_kernel_emu import FastKernelEmulator

HERE = os.path.dirname(os.path.abspath(__file__))
UNARY = ("tan", "cot", "asin", "acos", "atan")
TRIG_DOPS = ("TAN_F32", "COT_F32", "ASIN_F32", "ACOS_F32", "ATAN_F32", "ATAN2_F32", "ATAN2R_F32")
_lib = None


def lib():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="trig_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libtrig_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=gnu11", "-D_GNU_SOURCE", "-ffp-contract=off",
                               "-fno-math-errno", "-fPIC", "-shared", os.path.join(HERE, "trig_oracle.c"), "-o", so, "-lm"])
        _lib = ctypes.CDLL(so)
    return _lib


def _P(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def unary(name, x):
    """tan / cot / asin / acos / atan of the float32 array x, as the restatement computes it"""
    x = np.ascontiguousarray(x, np.float32); out = np.empty_like(x)
    lib().tr_unary_f32(UNARY.index(name), _P(x), _P(out), ctypes.c_size_t(len(x)))
    return out


def atan2(y, x):
    y, x = np.broadcast_arrays(np.asarray(y, np.float32), np.asarray(x, np.float32))
    y, x = np.ascontiguousarray(y), np.ascontiguousarray(x); out = np.empty_like(y)
    lib().tr_atan2_f32(_P(y), _P(x), _P(out), ctypes.c_size_t(len(y)))
    return out


def tancot_rcp(name, x, recip_kind):
    """tan / cot with the reciprocal computed as the correctly rounded float quotient (recip_kind 0) or the double
    quotient rounded to float (1); also returns the mask of elements that took the reciprocal branch"""
    x = np.ascontiguousarray(x, np.float32); out = np.empty_like(x); br = np.empty(len(x), np.int32)
    lib().tr_tancot_f32_rcp(int(name == "tan"), _P(x), _P(out), _P(br), int(recip_kind), ctypes.c_size_t(len(x)))
    return out, br.astype(bool)


def same_bits(a, b):
    """element-wise: the same bits, or both NaN (a NaN's payload is not part of the comparison: the GPU returns the
    canonical NaN where x86 propagates the operand's)"""
    a = np.asarray(a, np.float32); b = np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _trig(name, R, B):
    """the seven sweep operations on the accumulator bits R (and operand bits B); None for other names"""
    f = lambda v: np.ascontiguousarray(v).view(np.float32)
    if name in ("TAN_F32", "COT_F32", "ASIN_F32", "ACOS_F32", "ATAN_F32"):
        return unary(name[:-4].lower(), f(R)).view(np.uint32)
    if name == "ATAN2_F32":
        return atan2(f(R), f(B)).view(np.uint32)
    if name == "ATAN2R_F32":
        return atan2(f(B), f(R)).view(np.uint32)
    return None


class _TrigMixin:
    """Routes the trigonometric operations through the restatements: the interpreter hands every name that starts with
    CVT_ to _exec64 first, so their names are prefixed with CVT_ (in the lowered operation names too) and answered there."""
    def run(self, program):
        ren = lambda n: "CVT_" + n if n in TRIG_DOPS or (n.endswith("_U") and n[:-2] in TRIG_DOPS) else n
        program = dict(program, ops=[ren(n) for n in program["ops"]], fops=[ren(n) for n in program["fops"]])
        return super().run(program)

    def _exec64(self, name, imm, R, Rh, B, Bh, C, Ch, staged, cb):
        r = _trig(name[4:], R, B) if name.startswith("CVT_") else None
        return (r, Rh) if r is not None else super()._exec64(name, imm, R, Rh, B, Bh, C, Ch, staged, cb)


class TrigEmulator(_TrigMixin, Emulator):
    pass


class TrigKernelEmulator(_TrigMixin, FastKernelEmulator):
    """fast sweeps on the host-compiled kernel, the others on the interpreter"""
    pass
