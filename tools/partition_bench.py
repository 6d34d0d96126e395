"""Times ek_partition (virtual-call dispatch grouping) through the public C ABI only, for one or more builds of the
library, alternating between them case by case so that they share the machine's state.

    python tools/partition_bench.py enoki_b200/libenoki_b200.so other/libenoki_b200.so [--reps 20] [--json out.json]

Workload: n = 2^24 pointers (a render's ray count), K distinct 16-byte aligned pointers, assigned at random or in
coherent runs, plus one case above the device path's capacity.  Each timed call is the blocking ek_partition followed
by ek_sync (the device path returns with its last kernels queued); the median of --reps calls after --warmup calls is
reported, with GB/s against the algorithmic 12 B per element (8 B key read + 4 B index written).  The first call of
every case is also checked to give the same groups in every library."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

N = 1 << 24
GROUPS = [1, 4, 64, 256, 257, 4096, 65536]
FALLBACK_GROUPS = 65537
ALGO_BYTES = 12
# bytes per element the device path moves (ek_partition.cu): insert 8 + 4, count 4 + 4, then per radix pass the
# histogram and scatter reads plus the scatter writes, and 256 digit counts per 4096-element tile written, scanned
# (2 reads + 1 write) and read back by the scatter
SCAN_BYTES = 256 * 4 * 5 / 4096
DESIGN_BYTES = {1: 12 + 8 + 4 + 4 + 4 + SCAN_BYTES, 2: 12 + 8 + (4 + 4 + 8) + (8 + 8 + 4) + 2 * SCAN_BYTES}


def load(path):
    L = ctypes.CDLL(os.path.abspath(path))
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    L.ek_init.restype = ctypes.c_int
    L.ek_last_error.restype = ctypes.c_char_p
    L.ek_malloc.restype = vp
    L.ek_malloc.argtypes = [sz]
    L.ek_free.argtypes = [vp]
    L.ek_host_free.argtypes = [vp]
    L.ek_memcpy_to_device.argtypes = [vp, vp, sz]
    L.ek_memcpy_from_device.argtypes = [vp, vp, sz]
    L.ek_partition.restype = ctypes.c_int
    L.ek_partition.argtypes = [sz, vp, vp, vp, vp]
    assert L.ek_init() == 0, L.ek_last_error()
    return L


_libc = ctypes.CDLL(None)
_libc.free.argtypes = [ctypes.c_void_p]


def partition(L, keys_d, n, fetch):
    uniq, counts, lists = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    t0 = time.perf_counter()
    rc = L.ek_partition(n, keys_d, ctypes.byref(uniq), ctypes.byref(counts), ctypes.byref(lists))
    L.ek_sync()
    dt = time.perf_counter() - t0
    assert rc == 0, L.ek_last_error()
    k = ctypes.cast(counts, ctypes.POINTER(ctypes.c_uint32))[0]
    cnt = np.ctypeslib.as_array(ctypes.cast(counts, ctypes.POINTER(ctypes.c_uint32)), shape=(k + 1,))[1:].copy()
    ptrs = np.ctypeslib.as_array(ctypes.cast(lists, ctypes.POINTER(ctypes.c_uint64)), shape=(k,)).copy()
    result = None
    if fetch:
        un = np.ctypeslib.as_array(ctypes.cast(uniq, ctypes.POINTER(ctypes.c_uint64)), shape=(k,)).copy()
        idx = np.empty(n, np.uint32)
        off = 0
        for p, c in zip(ptrs, cnt):
            L.ek_memcpy_from_device(idx[off:].ctypes.data, int(p), int(c) * 4)
            off += int(c)
        result = (un, cnt, idx)
    for p in ptrs:
        L.ek_free(int(p))
    L.ek_host_free(uniq)
    L.ek_host_free(counts)
    _libc.free(lists)
    return dt, result


def make_keys(rng, k, coherent):
    cand = np.unique(rng.integers(1, 1 << 40, size=2 * k + 16, dtype=np.uint64))
    table = rng.permutation(cand)[:k] * np.uint64(16)
    if coherent:                                   # k runs of (almost) equal length, in a random order of the table
        return table[(np.arange(N, dtype=np.uint64) * np.uint64(k)) // np.uint64(N)]
    return table[rng.integers(0, k, N)]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                         # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--groups", type=int, nargs="+", default=GROUPS + [FALLBACK_GROUPS],
                    help="distinct pointer counts K (random and coherent assignment; random only above the capacity)")
    ap.add_argument("--json")
    a = ap.parse_args()
    libs = [load(p) for p in a.libs]
    print(f"card: {gpu_info()}", flush=True)
    print(f"n = {N}; algorithmic bytes/element = {ALGO_BYTES}; device path moves "
          f"{DESIGN_BYTES[1]:.1f} B/element with one radix pass (K <= 256), {DESIGN_BYTES[2]:.1f} with two", flush=True)
    cases = [(k, coh) for k in a.groups for coh in ((False, True) if k < FALLBACK_GROUPS else (False,))]
    rows = []
    rng = np.random.default_rng(2024)
    for k, coh in cases:
        keys = make_keys(rng, k, coh)
        bufs = []
        for L in libs:
            d = L.ek_malloc(N * 8)
            L.ek_memcpy_to_device(d, keys.ctypes.data, N * 8)
            bufs.append(d)
        first = [partition(L, d, N, True)[1] for L, d in zip(libs, bufs)]
        same = all(len(r[0]) == len(first[0][0]) and all((x == y).all() for x, y in zip(r, first[0])) for r in first[1:])
        times = [[] for _ in libs]
        for rep in range(a.warmup + a.reps):
            for j, (L, d) in enumerate(zip(libs, bufs)):
                dt, _ = partition(L, d, N, False)
                if rep >= a.warmup:
                    times[j].append(dt)
        for L, d in zip(libs, bufs):
            L.ek_free(d)
        row = {"K": k, "assignment": "coherent" if coh else "random", "same_result": bool(same),
               "ms": [float(np.median(t)) * 1e3 for t in times]}
        row["GBps_algorithmic"] = [ALGO_BYTES * N / (ms * 1e-3) / 1e9 for ms in row["ms"]]
        rows.append(row)
        print(f"K={k:6d} {row['assignment']:8s} " + "  ".join(
            f"[{j}] {ms:9.3f} ms {gb:7.2f} GB/s" for j, (ms, gb) in enumerate(zip(row["ms"], row["GBps_algorithmic"])))
            + ("" if same else "  RESULTS DIFFER"), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": gpu_info(), "n": N, "libs": a.libs, "design_bytes": DESIGN_BYTES, "rows": rows}, f, indent=1)
    return 0 if all(r["same_result"] for r in rows) else 1


if __name__ == "__main__":
    sys.exit(main())
