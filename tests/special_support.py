"""TEST INFRASTRUCTURE for the special functions erf, erfc, erfinv, lgamma and tgamma (EK_OP_ERF ... EK_OP_TGAMMA): the
plain-C restatements of tests/special_oracle.c, compiled into a temporary directory, and the numpy interpreter of
tests/ek_emulator.py taught the five new sweep operations through them (together with the hyperbolic ones of
tests/hyp_support.py and the trigonometric ones of tests/trig_support.py)."""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

import hyp_support as hs
import trig_support as ts
from ek_emulator import Emulator
from fast_kernel_emu import FastKernelEmulator

HERE = os.path.dirname(os.path.abspath(__file__))
UNARY = ("erf", "erfc", "erfinv", "lgamma", "tgamma")
SPEC_DOPS = tuple(n.upper() + "_F32" for n in UNARY)
_lib = None


def lib():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="special_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libspecial_oracle.so")
        oracle = os.path.join(os.path.dirname(HERE), "oracle")            # exp / log / sin: liboracle.so's or_*
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=gnu11", "-D_GNU_SOURCE", "-ffp-contract=off",
                               "-fno-math-errno", "-fPIC", "-shared", os.path.join(HERE, "special_oracle.c"), "-o", so,
                               "-L" + oracle, "-loracle", "-Wl,-rpath," + oracle, "-lm"])
        _lib = ctypes.CDLL(so)
    return _lib


def unary(name, x):
    """erf ... tgamma of the float32 array x, as the restatement computes it"""
    x = np.ascontiguousarray(x, np.float32); out = np.empty_like(x)
    lib().sp_unary_f32(UNARY.index(name), x.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p),
                       ctypes.c_size_t(len(x)))
    return out


same_bits = ts.same_bits


class _SpecMixin:
    """Routes the special functions through the restatements, the way hyp_support._HypMixin routes the hyperbolic
    ones: renamed with a CVT_ prefix, they reach _exec64 first."""
    def run(self, program):
        ren = lambda n: "CVT_" + n if n in SPEC_DOPS else n
        program = dict(program, ops=[ren(n) for n in program["ops"]], fops=[ren(n) for n in program["fops"]])
        return super().run(program)

    def _exec64(self, name, imm, R, Rh, B, Bh, C, Ch, staged, cb):
        if name.startswith("CVT_") and name[4:] in SPEC_DOPS:
            return unary(name[4:-4].lower(), np.ascontiguousarray(R).view(np.float32)).view(np.uint32), Rh
        return super()._exec64(name, imm, R, Rh, B, Bh, C, Ch, staged, cb)


class SpecEmulator(_SpecMixin, hs._HypMixin, ts._TrigMixin, Emulator):
    pass


class SpecKernelEmulator(_SpecMixin, hs._HypMixin, ts._TrigMixin, FastKernelEmulator):
    """fast sweeps on the host-compiled kernel, the others on the interpreter"""
    pass
