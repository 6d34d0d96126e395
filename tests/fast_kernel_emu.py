"""Runs the sweeps that the launcher would give to the 32-bit fast kernel on the HOST-COMPILED kernel source
(tests/cpu_kernel: enoki_b200/csrc/ek_sweep_fast.cu built as host code, one POSIX thread per CUDA thread) and everything
else on the numpy interpreter.  TEST INFRASTRUCTURE: the fast kernel was written without GPU access; this is how its
control flow, operand addressing and case bodies get executed before a GPU sees them."""
import ctypes
import os
import subprocess

import numpy as np

from ek_emulator import Emulator, T_BOOL, T_FLOAT32, T_INT32, T_INT8, T_UINT32, T_UINT8

HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def emu_lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-s", "-C", os.path.join(HERE, "cpu_kernel")])
        _lib = ctypes.CDLL(os.path.join(HERE, "cpu_kernel", "libemu_fast.so"))
        vp, u32 = ctypes.c_void_p, ctypes.c_uint32
        _lib.emu_run_fast.restype = ctypes.c_int
        _lib.emu_run_fast.argtypes = [vp, u32, u32, u32, vp, u32, vp, u32, vp, vp, u32, vp, vp, vp, u32,
                                      u32, u32, u32, u32, u32, u32, u32, u32, u32, u32]
    return _lib


_DT = {T_FLOAT32: np.float32, T_INT32: np.int32, T_UINT32: np.uint32, T_BOOL: np.uint8, T_INT8: np.int8, T_UINT8: np.uint8}


class FastKernelEmulator(Emulator):
    max_grid = 3                # CTAs per launch (each CTA loops over several tiles, like the persistent grid on the device)
    native_sweeps = 0

    def run(self, program):
        names = program["ops"]
        self.fops = program["fops"]
        for sw in program["sweeps"]:
            if "fast" in sw and sw["n"] > 1:
                self._native(sw)
                FastKernelEmulator.native_sweeps += 1
            else:
                self._sweep(names, sw)

    def _native(self, sw):
        fast = sw["fast"]
        n, T = sw["n"], fast["T"]
        hold = []                                   # keeps every buffer alive until the launch returns

        def addr(a):
            assert a.flags["C_CONTIGUOUS"]
            hold.append(a)
            return a.ctypes.data

        def writable(var):
            a = self.vars[var]
            if not (a.flags["C_CONTIGUOUS"] and a.flags["WRITEABLE"] and a.flags["OWNDATA"]):
                a = np.array(a, copy=True)
                self.vars[var] = a
            return a

        argw = np.array(fast["argw"], dtype=np.uint32) if fast["argw"] else np.zeros(1, np.uint32)
        outs = {}
        for var, aw, nbytes, typ in sw["outputs"]:
            dt = _DT.get(typ)
            assert dt is not None, ("output type", typ)
            buf = np.zeros(max(nbytes // np.dtype(dt).itemsize, 1), dtype=dt)
            outs[var] = (buf, typ, aw)
        for aw, var, is_out, address in sw["ptr_fix"]:
            if is_out:
                p = addr(outs[var][0])
            else:
                v = var if var in self.vars else self.by_address.get(address)
                assert v is not None and v in self.vars, ("pointer argument without data", var, hex(address))
                p = addr(writable(v))
            argw[aw] = p & 0xffffffff
            argw[aw + 1] = p >> 32
        words = []
        for sec in ("init", "body", "fini"):
            for fop, fl, b, c, dst, aux, imm in fast[sec]:
                words += [fop | (fl << 16), b | (c << 16), dst | (aux << 16), imm]
        prog = np.array(words, dtype=np.uint32) if words else np.zeros(4, np.uint32)
        lits = np.array(sw["lits"], dtype=np.uint32) if sw["lits"] else np.zeros(1, np.uint32)
        sc_ptr = np.zeros(max(len(sw["scalars"]), 1), np.uint64); sc_typ = np.zeros(max(len(sw["scalars"]), 1), np.uint8)
        for k, (var, typ) in enumerate(sw["scalars"]):
            a = np.ascontiguousarray(self.vars[var]).reshape(-1)
            if a.dtype == np.bool_:
                a = a.view(np.uint8)
            sc_ptr[k] = addr(a); sc_typ[k] = typ
        st_ptr = np.zeros(max(len(sw["staged"]), 1), np.uint64)
        st_unit = np.zeros(max(len(sw["staged"]), 1), np.uint16); st_es = np.zeros(max(len(sw["staged"]), 1), np.uint8)
        for k, (var, unit, es) in enumerate(sw["staged"]):
            a = np.ascontiguousarray(self.vars[var])
            if a.dtype == np.bool_:
                a = a.view(np.uint8)
            assert a.size == n and a.dtype.itemsize == es, (var, a.size, n, a.dtype, es)
            st_ptr[k] = addr(a); st_unit[k] = unit; st_es[k] = es
        n_tiles = (n + T * 16 - 1) // (T * 16)
        grid = max(1, min(n_tiles, self.max_grid))
        P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        rc = emu_lib().emu_run_fast(P(prog), len(fast["init"]), len(fast["body"]), len(fast["fini"]),
                                    P(lits), len(sw["lits"]), P(argw), len(fast["argw"]),
                                    P(sc_ptr), P(sc_typ), len(sw["scalars"]),
                                    P(st_ptr), P(st_unit), P(st_es), len(sw["staged"]),
                                    n, T, fast["n_tmp"], fast["n_in_units"], fast["off_bar"], fast["off_extra"], fast["off_slots"],
                                    fast["smem"], grid, fast["n_red"])
        assert rc == 0, ("emu_run_fast", rc)
        rfin = self.fops.index("RFIN")
        red_aw = {t[4] - len(sw["lits"]) for t in fast["fini"] if t[0] == rfin}      # dst = pool index of the result pointer
        for var, (buf, typ, aw) in outs.items():
            size = 1 if aw in red_aw else n         # reductions write one value into an 8-byte buffer
            v = buf[:size].copy()
            self.vars[var] = v.view(np.bool_) if typ == T_BOOL else v
        del hold
