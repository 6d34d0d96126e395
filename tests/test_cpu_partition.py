"""CPU: the kernels of enoki_b200/csrc/ek_partition.cu compiled as host code (tests/cpu_kernel/emu_partition.cpp, one
POSIX thread per CUDA thread, CTAs one after the other), driven through the same steps as ek_partition's host side:
hash insert + count, read back K / keys / counts, sort, id -> rank map, one or two radix passes with the scan done here.
Every result is checked against np.unique and a stable argsort."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def emu():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-s", "-C", os.path.join(HERE, "cpu_kernel"), "-f", "partition.mk"])
        _lib = ctypes.CDLL(os.path.join(HERE, "cpu_kernel", "libemu_partition.so"))
        vp, u32, u64, i32 = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_int
        _lib.emu_part_insert.argtypes = [vp, u64, u32, vp, vp, vp, vp, vp, vp]
        _lib.emu_part_hist.argtypes = [i32, vp, vp, vp, u64, u32, vp, u32]
        _lib.emu_part_scatter.argtypes = [i32, i32, vp, vp, vp, u64, u32, vp, u32, vp, vp, vp]
    return _lib


def P(a):
    return ctypes.c_void_p(a.ctypes.data) if a is not None else None


def constants():
    c = np.zeros(5, np.uint32)
    emu().emu_part_constants(P(c))
    return dict(zip(["threads", "max_groups", "slots", "count_bins", "tile"], (int(v) for v in c)))


def run_partition(keys, grid=3):
    """Returns (unique keys, counts, [index lists]) or None when the table overflowed."""
    L, C = emu(), constants()
    keys = np.ascontiguousarray(keys, np.uint64)
    n = len(keys)
    ids = np.full(n, 0xDEADBEEF, np.uint32)
    table = np.full(C["slots"], ~np.uint64(0), np.uint64)
    slot_id = np.full(C["slots"] + 1, 0xDEADBEEF, np.uint32)
    id_key = np.zeros(C["max_groups"], np.uint64)
    hdr = np.zeros(4, np.uint32)
    counts = np.zeros(C["max_groups"], np.uint32)
    assert L.emu_part_insert(P(keys), n, grid, P(ids), P(table), P(slot_id), P(id_key), P(hdr), P(counts)) == 0
    if hdr[1]:
        return None
    K = int(hdr[0])
    by_rank = np.argsort(id_key[:K], kind="stable")
    id_rank = np.empty(K, np.uint32)
    id_rank[by_rank] = np.arange(K, dtype=np.uint32)
    cnt = counts[:K][by_rank]
    start = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.uint32)
    lists = [np.full(int(c) + 4, 0xFFFFFFFF, np.uint32) for c in cnt]          # 4 guard words past every list
    list_ptrs = np.array([a.ctypes.data for a in lists], np.uint64)
    n_tiles = (n + C["tile"] - 1) // C["tile"]
    hist = np.zeros(256 * n_tiles, np.uint32)
    passes = 1 if K <= 256 else 2
    pairs = [np.zeros(n, np.uint64) for _ in range(2)]
    for p in range(passes):
        first, last = p == 0, p == passes - 1
        src = None if first else pairs[0]
        assert L.emu_part_hist(first, P(ids), P(src), P(id_rank), n, 8 * p, P(hist), n_tiles) == 0
        incl = np.cumsum(hist, dtype=np.uint64).astype(np.uint32)
        assert L.emu_part_scatter(first, last, P(ids), P(src), P(id_rank), n, 8 * p, P(incl), n_tiles,
                                  P(pairs[0]) if not last else None, P(list_ptrs) if last else None,
                                  P(start) if last else None) == 0
    for a, c in zip(lists, cnt):
        assert (a[int(c):] == 0xFFFFFFFF).all(), "scatter wrote past the end of a list"
    return id_key[:K][by_rank], cnt, [a[:int(c)] for a, c in zip(lists, cnt)]


def check(keys, grid=3):
    keys = np.asarray(keys, np.uint64)
    got = run_partition(keys, grid)
    assert got is not None, "unexpected overflow"
    uniq, cnt, lists = got
    want_u, want_c = np.unique(keys, return_counts=True)
    assert len(uniq) == len(want_u)
    assert (uniq == want_u).all() and (cnt == want_c).all()
    order = np.argsort(keys, kind="stable").astype(np.uint32)
    assert (np.concatenate(lists) == order).all()


def table(rng, k):
    cand = np.unique(rng.integers(1, 1 << 40, size=4 * k + 16, dtype=np.uint64))
    return np.sort(rng.permutation(cand)[:k]) * np.uint64(16)


@pytest.mark.parametrize("n,k", [(1, 1), (31, 3), (33, 2), (4095, 7), (4097, 256), (9000, 257), (20_000, 300)])
def test_random_assignment(n, k):
    rng = np.random.default_rng(n * 7 + k)
    t = table(rng, k)
    check(t[rng.integers(0, k, n)] if n >= k else t[:n])


def test_special_keys_and_runs():
    """0, 1, 2^63 - 1, 2^63, ~0, keys that differ only in the high 32 bits, multiples of 2^20, in long sorted runs."""
    rng = np.random.default_rng(5)
    special = np.array([0, 1, (1 << 63) - 1, 1 << 63, (1 << 64) - 1, 7 << 32, 9 << 32, 1 << 20, 3 << 20], np.uint64)
    check(np.repeat(special, 700))
    check(special[rng.integers(0, len(special), 6000)])
    check(np.full(5000, ~np.uint64(0), np.uint64))
    check(np.where(np.arange(6001) % 2 == 0, np.uint64(0), ~np.uint64(0)))
    check(np.arange(1, 260, dtype=np.uint64) << np.uint64(20))          # 259 keys: two passes, hash of aligned keys


def test_two_passes_many_groups():
    rng = np.random.default_rng(9)
    k = 1100
    check(table(rng, k)[rng.integers(0, k, 18_000)], grid=5)


def test_overflow_flag():
    """More distinct keys than the device path holds: the flag is set and the host falls back to its sort."""
    C = constants()
    k = C["max_groups"] + 1
    keys = (np.arange(k, dtype=np.uint64) + np.uint64(1)) * np.uint64(16)
    assert run_partition(keys, grid=4) is None
