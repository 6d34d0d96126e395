"""C2 with Float16 storage against C2 with Float32 storage, on both sweep kernels.

C2 (bench.py) reads four inputs and writes one output per element: 20 B with Float32 storage, 10 B with Float16 storage
(inputs widened to Float32, the expression computed in Float32, the result rounded to Float16).  The script times one
sweep of each variant at --n elements per launch with CUDA events around each launch (ek_set_timing), after a warm-up,
alternating the four variants (storage x kernel: the fast kernel, and the general kernel with ek_set_fast_mode(0)) rep
by rep.  The card's name and power limit are read in the same run; every output is checked against a host reference
(the C oracle's C2 on the same values, rounded to Float16 for Float16 storage).  Prints one JSON line and writes it to
--out when given.

    python tools/f16_probe.py [--n 67108864] [--reps 20] [--warmup 3] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    if q.returncode != 0:
        raise SystemExit("f16_probe: nvidia-smi failed -- this script measures on the GPU only")
    name, power, clock = (s.strip() for s in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def c2(ek, xs, f16):
    x0, x1, x2, x3 = (ek.Float32(x) for x in xs) if f16 else xs
    t = ek.fmadd(x0, x1, x2)
    r = ek.fmadd(ek.sin(ek.fmadd(x3, ek.exp(-(t * t)), x0)), x1, ek.sqrt(abs(t)))
    return ek.Float16(r) if f16 else r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 26)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()

    import enoki_b200 as ek
    if ek.device_count() == 0:
        raise SystemExit("f16_probe: no CUDA device")
    L = ek.lib()
    oracle = ctypes.CDLL(os.path.join(ROOT, "oracle", "liboracle.so"))
    info = card()
    n = args.n
    rng = np.random.default_rng(2)
    h = [rng.uniform(-4, 4, n).astype(np.float16) for _ in range(4)]
    f = [x.astype(np.float32) for x in h]          # the same values in both storages
    inputs = {True: [ek.Float16.copy(x) for x in h], False: [ek.Float32.copy(x) for x in f]}
    ref32 = np.zeros(n, np.float32)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    oracle.or_c2(P(f[0]), P(f[1]), P(f[2]), P(f[3]), P(ref32), ctypes.c_size_t(n))
    want = {False: ref32.view(np.uint32), True: ref32.astype(np.float16).view(np.uint16)}

    variants = [(f16, fast) for fast in (1, 0) for f16 in (False, True)]
    times = {v: [] for v in variants}
    checked = {}
    for rep in range(args.warmup + args.reps):
        for f16, fast in variants:
            L.ek_set_fast_mode(fast)
            L.ek_set_timing(1)
            L.ek_stats_reset()
            out = c2(ek, inputs[f16], f16)
            out.eval()
            ek.cuda_sync()
            st = ek.stats()
            L.ek_set_timing(0)
            assert int(st.sweep_launches) == 1, ("one sweep per C2", int(st.sweep_launches))
            assert (int(st.fast_launches) == 1) == bool(fast), ("kernel", fast, int(st.fast_launches))
            if rep >= args.warmup:
                times[(f16, fast)].append(float(st.last_kernel_ms))
            if (f16, fast) not in checked:
                got = out.numpy()
                got = got.view(np.uint16 if f16 else np.uint32)
                checked[(f16, fast)] = int((got != want[f16]).sum())
            del out
    L.ek_set_fast_mode(1)

    res = {"workload": f"C2 at n = {n}", "card": info, "reps": args.reps, "variants": []}
    for f16, fast in variants:
        t = np.array(times[(f16, fast)])
        bpe = 10 if f16 else 20
        med = float(np.median(t))
        res["variants"].append({"storage": "float16" if f16 else "float32", "kernel": "fast" if fast else "general",
                                "bytes_per_elem": bpe, "kernel_ms_median": med, "kernel_ms_min": float(t.min()),
                                "kernel_ms_max": float(t.max()), "gb_per_s": bpe * n / (med * 1e-3) / 1e9,
                                "mismatches_vs_host": checked[(f16, fast)]})
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    if any(v["mismatches_vs_host"] for v in res["variants"]):
        raise SystemExit("f16_probe: an output differs from the host reference")


if __name__ == "__main__":
    main()
