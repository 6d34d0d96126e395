"""Generate tests/golden/hyp.npz from the reference's single precision sinh, cosh, tanh, asinh, acosh, atanh, cbrt and
sincosh (the AVX2 Packet<float, 8> CPU path, compiled from tests/golden/ref_hyp.cpp into a temporary directory), and
tests/golden/hyp_traced.json, the dry run of the same functions' generic bodies recorded one primitive at a time on a
CUDAArray<float> (tests/golden/ref_hyp_traced.cpp over libenoki_b200.so; nothing is launched).  Run in the dev
container, where the reference lies (REF, default /root/reference), after build(); both files are committed.

    python tests/golden/make_golden_hyp.py

hyp.npz: `x` (special values -- signed zeros, denormals, +-1, the branch thresholds of every function and their
neighbours, values near the exp overflow, 1e10 and its neighbours, infinities, NaNs -- and random values over the whole
range, over [-1.2, 1.2] and over [-20, 20]) with `sinh`, `cosh`, `tanh`, `asinh`, `acosh`, `atanh`, `cbrt`, `sincosh_s`,
`sincosh_c`.
hyp_traced.json: {name: {"x": input variable, "out": [result variables], "plan": listing, "program": program}}.
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
NAMES = ("sinh", "cosh", "tanh", "asinh", "acosh", "atanh", "cbrt", "sincosh_s", "sincosh_c")


def special_f32():
    """Signed zeros, the smallest / largest denormals and normals, 1e-45 ... 1e-30, +-1 and the thresholds of every
    function (sinh 1, tanh 0.625, asinh 0.51 and 1e10, acosh 1.49 and 1e10 + 1, atanh 0.5 and 1) with their float
    neighbours, the exp overflow and underflow bounds (+-88.3762588501, and 44.19 for tanh's exp(2x)), large values,
    infinities, and NaNs with and without a payload."""
    base = np.array([0.0, 1e-45, 1.1754942e-38, 1.17549435e-38, 1e-30, 1e-10, 1e-4, 0.25, 0.5, 0.51, 0.625, 1.0, 1.49, 1.5,
                     2.0, 3.0, 8.0, 27.0, 44.0, 44.1881294, 44.19, 88.0, 88.3762588501, 88.5, 89.0, 100.0, 1e10,
                     1e10 + 1, 1e20, 3.4028235e38], np.float32).view(np.uint32)
    v = np.concatenate([base, base - 1, base + 1, np.array([0x7f800000, 0x7fc00000, 0x7fa00000, 0x7fffffff, 0x007fffff,
                                                           0x00000001, 0x00000002], np.uint32)])
    return np.concatenate([v, v | np.uint32(0x80000000)]).view(np.float32)


def traced():
    """tests/golden/ref_hyp_traced.cpp, compiled against this repository's headers and library, and its output"""
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "ref_hyp_traced")
        lib = os.path.join(ROOT, "enoki_b200")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-w", "-fno-strict-aliasing", *ISA, "-ffp-contract=off",
                               "-DENOKI_CUDA=1", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(REF, "include"),
                               os.path.join(HERE, "ref_hyp_traced.cpp"), "-o", exe, "-L" + lib, "-lenoki_b200",
                               "-Wl,-rpath," + lib, "-L/usr/local/cuda/lib64", "-lcudart"])
        return json.loads(subprocess.run([exe], capture_output=True, text=True, check=True).stdout)


def main():
    rng = np.random.default_rng(20261018)
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "libref_hyp.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", *ISA, "-ffp-contract=off", "-fno-math-errno", "-fPIC",
                               "-shared", "-w", "-I" + os.path.join(REF, "include"), os.path.join(HERE, "ref_hyp.cpp"),
                               "-o", so])
        L = ctypes.CDLL(so)
        x = np.concatenate([special_f32(), rng.integers(0, 1 << 32, 6000, dtype=np.uint64).astype(np.uint32).view(np.float32),
                            rng.uniform(-1.2, 1.2, 4000).astype(np.float32), rng.uniform(-20.0, 20.0, 4000).astype(np.float32)])
        x = np.concatenate([x, np.zeros((-len(x)) % 8, np.float32)])
        d = {"x": x}
        for which, name in enumerate(NAMES):
            out = np.zeros_like(x)
            L.ref_hyp_unary(which, P(x), P(out), ctypes.c_size_t(len(x)))
            d[name] = out
    np.savez_compressed(os.path.join(HERE, "hyp.npz"), **d)
    print("wrote", os.path.join(HERE, "hyp.npz"), {k: v.shape for k, v in d.items()})
    with open(os.path.join(HERE, "hyp_traced.json"), "w") as f:
        json.dump(traced(), f, separators=(",", ":"))
        f.write("\n")
    print("wrote", os.path.join(HERE, "hyp_traced.json"))


if __name__ == "__main__":
    main()
