"""Generate tests/golden/convert_f16.npz from the reference's half (include/enoki/half.h with F16C, compiled from
tests/golden/ref_half.cpp into a temporary directory) and the unmodified reference CPU path (oracle/_ref/libenoki_ref.so,
`make -C oracle ref`).  Run in the dev container, where the reference lies (REF, default /root/reference); the .npz is
committed.

    python tests/golden/make_golden_f16.py
"""
import ctypes
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import CONVERT_DTYPES, CONVERT_TYPES, P, R, SZ, convert_inputs  # noqa: E402

REF = os.environ.get("REF", "/root/reference")


def half_lib(tmp):
    so = os.path.join(tmp, "libref_half.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-mavx2", "-mfma", "-mf16c", "-fPIC", "-shared", "-w",
                           "-I" + os.path.join(REF, "include"), os.path.join(HERE, "ref_half.cpp"), "-o", so])
    return ctypes.CDLL(so)


def f16_rounding_boundaries(step=1):
    """Float32 bit patterns around the rounding boundaries of binary16 (those after every `step`-th half), both signs:
    the midpoint to the next half and the floats just below / above it, the half itself, the overflow threshold 65520,
    the subnormal range and its lower end 2^-25, zeros, infinities and NaNs with several payloads."""
    h = np.concatenate([np.arange(0, 0x7c00, step), [0x3ff, 0x400, 0x7bff]]).astype(np.uint32)
    lo = h.astype(np.uint16).view(np.float16).astype(np.float32).view(np.uint32).astype(np.uint64)
    hi = (h + 1).astype(np.uint16).view(np.float16).astype(np.float32).view(np.uint32).astype(np.uint64)
    mid = (lo + hi) // 2
    extra = [0x477fe000, 0x477fefff, 0x477ff000, 0x477ff001, 0x7f7fffff, 0x7f800000, 0x00000001, 0x00800000, 0x32ffffff,
             0x33000000, 0x33000001, 0x33800000, 0x387fc000, 0x387fe000, 0x38800000, 0x7f800001, 0x7fc00000, 0x7fe00000,
             0x7fffffff, 0x7fa00000, 0x7f802000]
    v = np.concatenate([mid - 1, mid, mid + 1, lo, np.array(extra, np.uint64)]).astype(np.uint32)
    return np.concatenate([v, v | np.uint32(0x80000000)]).view(np.float32)


def convert_f16(H):
    """Every binary16 bit pattern converted to the ten numeric types (half_<dst>_<mode>; mode 1 / 2 = floor2int /
    ceil2int, to Int32): the half widened to float (half.h), then the reference's Float32 conversion -- and the ten
    types converted to half (<src>_half) on the inputs of convert.npz plus, for Float32, the rounding boundaries of every
    7th half and for Float64 the values where rounding twice (through Float32) differs from rounding once."""
    rng = np.random.default_rng(16)
    d = {"x_half": np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)}
    f = np.zeros(1 << 16, np.float32)
    H.ref_half_to_float(P(d["x_half"]), P(f), SZ(1 << 16))
    for dst, dc in CONVERT_TYPES.items():
        for mode in ((0, 1, 2) if dst == "Int32" else (0,)):
            out = np.zeros(1 << 16, CONVERT_DTYPES[dst])
            assert R.ref_convert(10, dc, mode, P(f), P(out), SZ(1 << 16)) == 0, (dst, mode)
            d[f"half_{dst}_{mode}"] = out
    for src, sc in CONVERT_TYPES.items():
        x = convert_inputs(rng, src)
        if src == "Float32":
            x = np.concatenate([x, f16_rounding_boundaries(step=7)])
        if src == "Float64":      # 1 + 2^-11 (+ 2^-30): a tie of the half grid that only the double rounding sees
            x = np.concatenate([x, [1 + 2.0 ** -11 + 2.0 ** -30, 1 + 2.0 ** -11 - 2.0 ** -30, 65519.99999, 2.0 ** -25 * (1 + 2.0 ** -40)]])
        x = np.ascontiguousarray(x, CONVERT_DTYPES[src])
        out = np.zeros(len(x), np.uint16)
        assert H.ref_half_from(sc, P(x), P(out), SZ(len(x))) == 0, src
        d[f"x_{src}"] = x
        d[f"{src}_half"] = out
    np.savez_compressed(os.path.join(HERE, "convert_f16.npz"), **d)


if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as tmp:
        convert_f16(half_lib(tmp))
    print("convert_f16.npz written to", HERE)
