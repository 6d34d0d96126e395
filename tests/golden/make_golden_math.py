"""Generate tests/golden/math.npz from the reference's single precision pow, frexp, hypot, dawson and erfi
(the AVX2 Packet<float, 8> CPU path, compiled from tests/golden/ref_math.cpp into a temporary directory), and
tests/golden/math_traced.json, the dry run of the same functions' generic bodies recorded one primitive at a time on
CUDAArray<float> arrays (tests/golden/ref_math_traced.cpp over libenoki_b200.so; nothing is launched).  Run in the dev
container, where the reference lies (REF, default /root/reference), after build(); both files are committed.

    python tests/golden/make_golden_math.py

math.npz: `x` (special values, thresholds and random values) with `frexp_m`, `frexp_e`, `dawson`, `erfi`; `bx`, `by`
(pairs: the cross product of the special values, random bit patterns, positive bases with exponents in [-8, 8] and
equal magnitudes) with `pow`, `hypot`.
math_traced.json: {name: {"x": input variable, "y": second input (binary), "out": [results], "plan": listing,
"program": program}}.
"""
import ctypes
import json
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("REF", "/root/reference")
P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
ISA = ["-mavx2", "-mfma", "-mf16c", "-mbmi", "-mbmi2", "-mlzcnt"]
BINARY = ("pow", "hypot")
UNARY = ("frexp_m", "frexp_e", "dawson", "erfi")


def specials():
    """signed zeros, denormals, the smallest / largest normals, +-1 and its neighbours, small integers, large values,
    infinities and NaNs with and without a payload"""
    pos = np.array([0.0, 1e-45, 1e-40, 1.1754942e-38, 1.17549435e-38, 1e-30, 1e-4, 0.5, 0.99999994, 1.0, 1.0000001, 1.5,
                    2.0, 2.5, 3.0, 7.0, 8.0, 10.0, 88.0, 100.0, 127.0, 128.0, 1e10, 16777216.0, 3.4028235e38], np.float32)
    nan_inf = np.array([0x7f800000, 0x7fc00000, 0x7fa00000, 0x7fffffff], np.uint32).view(np.float32)
    pos = np.concatenate([pos, nan_inf])
    return np.concatenate([pos, -pos])


def unary_inputs(rng):
    return np.concatenate([specials(), rng.integers(0, 1 << 32, 3000, dtype=np.uint64).astype(np.uint32).view(np.float32),
                           rng.uniform(-4, 4, 1500).astype(np.float32), rng.uniform(-12, 12, 1500).astype(np.float32)])


def binary_inputs(rng):
    s = specials()
    cx, cy = np.meshgrid(s, s)
    bits = lambda n: rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
    n = 1200
    base = rng.uniform(0, 10, n).astype(np.float32); ex = rng.uniform(-8, 8, n).astype(np.float32)
    eq = rng.uniform(-1e3, 1e3, n).astype(np.float32)
    x = np.concatenate([cx.ravel(), bits(3000), base, eq])
    y = np.concatenate([cy.ravel(), bits(3000), ex, -eq])
    return x, y


def traced():
    """tests/golden/ref_math_traced.cpp, compiled against this repository's headers and library, and its output"""
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "ref_math_traced")
        lib = os.path.join(ROOT, "enoki_b200")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-w", "-fno-strict-aliasing", *ISA, "-ffp-contract=off",
                               "-DENOKI_CUDA=1", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(REF, "include"),
                               os.path.join(HERE, "ref_math_traced.cpp"), "-o", exe, "-L" + lib, "-lenoki_b200",
                               "-Wl,-rpath," + lib, "-L/usr/local/cuda/lib64", "-lcudart"])
        return json.loads(subprocess.run([exe], capture_output=True, text=True, check=True).stdout)


def pad8(a):
    return np.concatenate([a, np.zeros((-len(a)) % 8, np.float32)])


def main():
    rng = np.random.default_rng(20261020)
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "libref_math.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", *ISA, "-ffp-contract=off", "-fno-math-errno", "-fPIC",
                               "-shared", "-w", "-I" + os.path.join(REF, "include"), os.path.join(HERE, "ref_math.cpp"),
                               "-o", so])
        L = ctypes.CDLL(so)
        x = pad8(unary_inputs(rng))
        bx, by = (pad8(v) for v in binary_inputs(rng))
        d = {"x": x, "bx": bx, "by": by}
        for which, name in enumerate(UNARY):
            out = np.zeros_like(x)
            L.ref_math_unary(which, P(x), P(out), ctypes.c_size_t(len(x)))
            d[name] = out
        for which, name in enumerate(BINARY):
            out = np.zeros_like(bx)
            L.ref_math_binary(which, P(bx), P(by), P(out), ctypes.c_size_t(len(bx)))
            d[name] = out
    np.savez_compressed(os.path.join(HERE, "math.npz"), **d)
    print("wrote", os.path.join(HERE, "math.npz"), {k: v.shape for k, v in d.items()})
    with open(os.path.join(HERE, "math_traced.json"), "w") as f:
        json.dump(traced(), f, separators=(",", ":"))
        f.write("\n")
    print("wrote", os.path.join(HERE, "math_traced.json"))


if __name__ == "__main__":
    main()
