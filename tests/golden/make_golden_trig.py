"""Generate tests/golden/trig.npz from the reference's single precision tan, cot, asin, acos, atan and atan2 (the AVX2
Packet<float, 8> CPU path, compiled from tests/golden/ref_trig.cpp into a temporary directory).  Run in the dev
container, where the reference lies (REF, default /root/reference); the .npz is committed.

    python tests/golden/make_golden_trig.py

Contents: `x` (special values, the tan / cot branch points k pi / 4 and their neighbours, and random values over the
whole range and over [-1, 1]) with `tan`, `cot`, `asin`, `acos`, `atan`; `y2`, `x2` (the cross product of special
values -- signed zeros, denormals, +-1, infinities, NaN, |y| = |x| -- and random pairs) with `atan2`.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("REF", "/root/reference")
P = lambda a: a.ctypes.data_as(ctypes.c_void_p)


def special_f32():
    """Signed zeros, the smallest / largest denormals and normals, +-1, the asin / acos branch point 0.5, infinities and
    NaNs with and without a payload, and values where tan / cot change branch (k pi / 4) with their neighbours."""
    bits = [0x00000000, 0x00000001, 0x007fffff, 0x00800000, 0x3f800000, 0x3f000000, 0x3effffff, 0x3f000001, 0x3f7fffff,
            0x3f800001, 0x7f7fffff, 0x7f800000, 0x7fc00000, 0x7fa00000, 0x7fffffff, 0x38d1b717, 0x38d1b716, 0x4f000000,
            0x4effffff, 0x4b800000]
    v = np.array(bits, np.uint32)
    k = np.arange(1, 64, dtype=np.float64)
    br = (k * np.pi / 4).astype(np.float32).view(np.uint32)
    v = np.concatenate([v, br - 1, br, br + 1])
    return np.concatenate([v, v | np.uint32(0x80000000)]).view(np.float32)


def atan2_specials():
    s = np.array([0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, -1.1754942e-38, 1.0, -1.0, 0.5, -2.0, 3.0, -3.0,
                  np.inf, -np.inf, np.nan, 3.4028235e38, -3.4028235e38], np.float32)
    y, x = np.meshgrid(s, s, indexing="ij")
    return y.ravel(), x.ravel()


def main():
    rng = np.random.default_rng(20261017)
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "libref_trig.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-mavx2", "-mfma", "-mf16c", "-mbmi", "-mbmi2", "-mlzcnt",
                               "-ffp-contract=off", "-fno-math-errno", "-fPIC", "-shared", "-w",
                               "-I" + os.path.join(REF, "include"), os.path.join(HERE, "ref_trig.cpp"), "-o", so])
        L = ctypes.CDLL(so)

        def pad8(a):
            return np.concatenate([a, np.zeros((-len(a)) % 8, a.dtype)])

        x = np.concatenate([special_f32(), rng.integers(0, 1 << 32, 6000, dtype=np.uint64).astype(np.uint32).view(np.float32),
                            rng.uniform(-1.0, 1.0, 3000).astype(np.float32), rng.uniform(-20.0, 20.0, 3000).astype(np.float32)])
        x = pad8(x)
        d = {"x": x}
        for which, name in enumerate(("tan", "cot", "asin", "acos", "atan")):
            out = np.zeros_like(x)
            L.ref_trig_unary(which, P(x), P(out), ctypes.c_size_t(len(x)))
            d[name] = out
        ys, xs = atan2_specials()
        ry = rng.integers(0, 1 << 32, 8000, dtype=np.uint64).astype(np.uint32).view(np.float32)
        rx = rng.integers(0, 1 << 32, 8000, dtype=np.uint64).astype(np.uint32).view(np.float32)
        uy = rng.uniform(-10, 10, 4000).astype(np.float32); ux = rng.uniform(-10, 10, 4000).astype(np.float32)
        y2 = pad8(np.concatenate([ys, ry, uy, ux])); x2 = pad8(np.concatenate([xs, rx, ux, -ux]))   # (|y| = |x| pairs last)
        out = np.zeros_like(y2)
        L.ref_trig_atan2(P(y2), P(x2), P(out), ctypes.c_size_t(len(y2)))
        d.update(y2=y2, x2=x2, atan2=out)
    np.savez_compressed(os.path.join(HERE, "trig.npz"), **d)
    print("wrote", os.path.join(HERE, "trig.npz"), {k: v.shape for k, v in d.items()})


if __name__ == "__main__":
    main()
