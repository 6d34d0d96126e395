"""Generate tests/golden/ell.npz from the reference's single precision carlson_rf, carlson_rd, carlson_rc,
comp_ellint_1 / 2 and ellint_1 / 2 (the AVX2 Packet<float, 8> CPU path, compiled from tests/golden/ref_ell.cpp into a
temporary directory), and tests/golden/ell_traced.json, the dry runs of one pass of each Carlson integral's duplication
loop and of its epilogue, recorded one primitive at a time on CUDAArray<float> arrays (tests/golden/ell_traced.cpp
over libenoki_b200.so; nothing is launched).  Run in the dev container, where the reference lies (REF, default
/root/reference), after build(); both files are committed.

    python tests/golden/make_golden_ell.py

ell.npz: `tx`, `ty`, `tz` (triples: special values, the convergence thresholds and their neighbours, valid random triples
over 2^-40 ... 2^40) with `carlson_rf`, `carlson_rd`; `px`, `py` (pairs, the same kinds) with `carlson_rc`; `k` with
`comp_ellint_1`, `comp_ellint_2`; `phi`, `kk` with `ellint_1`, `ellint_2`.  special.h's k is squared: K(k) = R_F(0, 1 - k^2,
1).
ell_traced.json: {name: {"in": {role: variable}, "out": {role: variable}, "plan": listing, "program": program}}.
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
# the loop thresholds of special.h rounded to float (rf, rd, rc: eps^(1/6), * 0.6, * 0.48)
THRESHOLDS = np.array([0.070154, 0.070154 * 0.6, 0.070154 * 0.48], np.float32)


def specials():
    """valid argument values: zero (x only), denormals, tiny and huge normals, 1 and its neighbours, small integers"""
    return np.array([0.0, 1e-45, 1e-40, 1.17549435e-38, 1e-30, 1e-12, 1e-4, 0.25, 0.5, 0.99999994, 1.0, 1.0000001, 2.0,
                     3.0, 10.0, 1e4, 1e12, 1e30, 3.4028235e38], np.float32)


def near_thresholds():
    """every threshold and its three neighbours on either side"""
    out = []
    for t in THRESHOLDS:
        v = t
        for _ in range(3):
            v = np.nextafter(v, np.float32(-np.inf))
        for _ in range(7):
            out.append(v)
            v = np.nextafter(v, np.float32(np.inf))
    return np.array(out, np.float32)


def triples(rng, n=6000):
    s = specials()
    pos = s[s > 0]
    cx, cy, cz = np.meshgrid(s, pos, pos, indexing="ij")
    t = near_thresholds()
    # mu = 1 and |X| = eps: x = 1 + e, y = 1 - e, z = 1
    tx, ty, tz = 1 + t, 1 - t, np.ones_like(t)
    lg = lambda m: np.exp2(rng.uniform(-40, 40, m)).astype(np.float32)
    rx, ry, rz = lg(n), lg(n), lg(n)
    rx[: n // 10] = 0
    x = np.concatenate([cx.ravel(), tx, rx]).astype(np.float32)
    y = np.concatenate([cy.ravel(), ty, ry]).astype(np.float32)
    z = np.concatenate([cz.ravel(), tz, rz]).astype(np.float32)
    return x, y, z


def pairs(rng, n=6000):
    s = specials()
    pos = s[s > 0]
    cx, cy = np.meshgrid(s, pos, indexing="ij")
    t = near_thresholds()
    lg = lambda m: np.exp2(rng.uniform(-40, 40, m)).astype(np.float32)
    rx, ry = lg(n), lg(n)
    rx[: n // 10] = 0
    x = np.concatenate([cx.ravel(), 1 + t, rx]).astype(np.float32)
    y = np.concatenate([cy.ravel(), 1 - t, ry]).astype(np.float32)
    return x, y


def traced():
    """tests/golden/ell_traced.cpp, compiled against this repository's headers and library, and its output"""
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "ell_traced")
        lib = os.path.join(ROOT, "enoki_b200")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-w", "-fno-strict-aliasing", *ISA, "-ffp-contract=off",
                               "-DENOKI_CUDA=1", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(REF, "include"),
                               os.path.join(HERE, "ell_traced.cpp"), "-o", exe, "-L" + lib, "-lenoki_b200",
                               "-Wl,-rpath," + lib, "-L/usr/local/cuda/lib64", "-lcudart"])
        return json.loads(subprocess.run([exe], capture_output=True, text=True, check=True).stdout)


def pad8(a):
    return np.concatenate([a, np.full((-len(a)) % 8, 1, np.float32)])


def main():
    rng = np.random.default_rng(20261018)
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "libref_ell.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", *ISA, "-ffp-contract=off", "-fno-math-errno", "-fPIC",
                               "-DNDEBUG", "-shared", "-w", "-I" + os.path.join(REF, "include"),
                               os.path.join(HERE, "ref_ell.cpp"), "-o", so])
        L = ctypes.CDLL(so)
        tx, ty, tz = (pad8(v) for v in triples(rng))
        px, py = (pad8(v) for v in pairs(rng))
        k = pad8(np.concatenate([np.array([0, 0.1, 0.5, 0.9, 0.99, 0.999999, -0.5, -0.99], np.float32),
                                 rng.uniform(-1, 1, 4000).astype(np.float32)]))
        phi = pad8(np.concatenate([np.array([0, 0.5, 1.5, 1.5707964, 3.0, -1.0, 10.0, -7.5], np.float32),
                                   rng.uniform(-8, 8, 4000).astype(np.float32)]))
        kk = pad8(np.concatenate([np.array([0.5, 0.9, 0.1, 0.99, 0.3, -0.7, 0.2, 0.0], np.float32),
                                  rng.uniform(-1, 1, 4000).astype(np.float32)]))
        d = {"tx": tx, "ty": ty, "tz": tz, "px": px, "py": py, "k": k, "phi": phi, "kk": kk}
        for which, name in enumerate(("carlson_rf", "carlson_rd")):
            out = np.zeros_like(tx)
            L.ref_ell_carlson(which, P(tx), P(ty), P(tz), P(out), ctypes.c_size_t(len(tx)))
            d[name] = out
        out = np.zeros_like(px)
        L.ref_ell_carlson(2, P(px), P(py), P(py), P(out), ctypes.c_size_t(len(px)))
        d["carlson_rc"] = out
        for which, name in enumerate(("comp_ellint_1", "comp_ellint_2")):
            out = np.zeros_like(k)
            L.ref_ell_integral(which, P(k), P(k), P(out), ctypes.c_size_t(len(k)))
            d[name] = out
        for which, name in enumerate(("ellint_1", "ellint_2")):
            out = np.zeros_like(phi)
            L.ref_ell_integral(2 + which, P(phi), P(kk), P(out), ctypes.c_size_t(len(phi)))
            d[name] = out
    np.savez_compressed(os.path.join(HERE, "ell.npz"), **d)
    print("wrote", os.path.join(HERE, "ell.npz"), {k_: v.shape for k_, v in d.items()})
    with open(os.path.join(HERE, "ell_traced.json"), "w") as f:
        json.dump(traced(), f, separators=(",", ":"))
        f.write("\n")
    print("wrote", os.path.join(HERE, "ell_traced.json"))


if __name__ == "__main__":
    main()
