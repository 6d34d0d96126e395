"""Generate tests/golden/special.npz from the reference's single precision erf, erfc, erfinv, lgamma and tgamma (the
AVX2 Packet<float, 8> CPU path, compiled from tests/golden/ref_special.cpp into a temporary directory), and
tests/golden/special_traced.json, the dry run of the same functions' generic bodies (and of the normal-sampling step
sqrt(2) * erfinv(2u - 1)) recorded one primitive at a time on a CUDAArray<float> (tests/golden/ref_special_traced.cpp
over libenoki_b200.so; nothing is launched).  Run in the dev container, where the reference lies (REF, default
/root/reference), after build(); both files are committed.

    python tests/golden/make_golden_special.py

special.npz: `x` (special values -- signed zeros, denormals, +-1 and its neighbours, the branch thresholds of every
function with their float neighbours, the non-positive integers, tgamma's exp overflow region, infinities, NaNs -- and
random values over the whole range, over [-3, 3], over [-1, 1] and over [-40, 40]) with `erf`, `erfc`, `erfinv`,
`lgamma`, `tgamma`.
special_traced.json: {name: {"x": input variable, "out": [result variable], "plan": listing, "program": program}}.
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
NAMES = ("erf", "erfc", "erfinv", "lgamma", "tgamma")


def neighbours(v, k):
    """the float32 values v and its k neighbours on either side, for each v"""
    b = np.asarray(v, np.float32).view(np.int32).astype(np.int64)
    return np.concatenate([b + d for d in range(-k, k + 1)]).astype(np.uint32).view(np.float32)


def special_f32():
    """Signed zeros, denormals, the smallest / largest normals, +-1 with 4 neighbours on either side; the thresholds of
    erf / erfc (|x| = 1 and 2), erfinv's w = 5 (|x| = sqrt(1 - e^-5)) and lgamma's 0.5, with 64, 64, 256 and 4
    neighbours; the non-positive integers down to -40 and a few large ones, with their neighbours; tgamma's exp overflow
    region (lgamma(x) = 88.38 near x = 35.04, and around 34 ... 36); large values, infinities and NaNs with and
    without a payload."""
    base = np.array([0.0, 1e-45, 1e-40, 1.1754942e-38, 1.17549435e-38, 1e-30, 1e-10, 1e-4, 0.25, 0.5, 0.75, 1.5, 3.0, 3.9,
                     4.0, 9.0, 10.0, 30.0, 100.0, 1e10, 1e20, 3.4028235e38], np.float32)
    thresholds = [neighbours([1.0, -1.0], 4), neighbours([2.0, -2.0], 64), neighbours([1.0, -1.0], 64),
                  neighbours(np.float32(np.sqrt(1 - np.exp(-5.0))) * np.float32([1, -1]), 256),
                  neighbours([0.5], 4)]
    ints = -np.arange(0, 41, dtype=np.float32)
    ints = np.concatenate([ints, np.float32([-100, -1000, -1e6, -8388608, -1e10])])
    overflow = np.concatenate([np.linspace(34.0, 36.0, 401, dtype=np.float32), neighbours([35.0400009], 64),
                               np.linspace(-36.0, -34.0, 201, dtype=np.float32)])
    nan_inf = np.array([0x7f800000, 0x7fc00000, 0x7fa00000, 0x7fffffff, 0x007fffff, 0x00000001], np.uint32).view(np.float32)
    pos = np.concatenate([base, nan_inf])
    return np.concatenate([pos, -pos, *thresholds, neighbours(ints, 2), overflow])


def traced():
    """tests/golden/ref_special_traced.cpp, compiled against this repository's headers and library, and its output"""
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "ref_special_traced")
        lib = os.path.join(ROOT, "enoki_b200")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-w", "-fno-strict-aliasing", *ISA, "-ffp-contract=off",
                               "-DENOKI_CUDA=1", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(REF, "include"),
                               os.path.join(HERE, "ref_special_traced.cpp"), "-o", exe, "-L" + lib, "-lenoki_b200",
                               "-Wl,-rpath," + lib, "-L/usr/local/cuda/lib64", "-lcudart"])
        return json.loads(subprocess.run([exe], capture_output=True, text=True, check=True).stdout)


def main():
    rng = np.random.default_rng(20261019)
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "libref_special.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", *ISA, "-ffp-contract=off", "-fno-math-errno", "-fPIC",
                               "-shared", "-w", "-I" + os.path.join(REF, "include"), os.path.join(HERE, "ref_special.cpp"),
                               "-o", so])
        L = ctypes.CDLL(so)
        x = np.concatenate([special_f32(), rng.integers(0, 1 << 32, 6000, dtype=np.uint64).astype(np.uint32).view(np.float32),
                            rng.uniform(-3.0, 3.0, 4000).astype(np.float32), rng.uniform(-1.0, 1.0, 4000).astype(np.float32),
                            rng.uniform(-40.0, 40.0, 4000).astype(np.float32)])
        x = np.concatenate([x, np.zeros((-len(x)) % 8, np.float32)])
        d = {"x": x}
        for which, name in enumerate(NAMES):
            out = np.zeros_like(x)
            L.ref_special_unary(which, P(x), P(out), ctypes.c_size_t(len(x)))
            d[name] = out
    np.savez_compressed(os.path.join(HERE, "special.npz"), **d)
    print("wrote", os.path.join(HERE, "special.npz"), {k: v.shape for k, v in d.items()})
    with open(os.path.join(HERE, "special_traced.json"), "w") as f:
        json.dump(traced(), f, separators=(",", ":"))
        f.write("\n")
    print("wrote", os.path.join(HERE, "special_traced.json"))


if __name__ == "__main__":
    main()
