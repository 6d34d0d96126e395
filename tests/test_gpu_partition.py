"""ek_partition (virtual-call dispatch grouping, ek_partition.cu) on the GPU, checked exactly against np.unique and a stable
argsort: sizes around the warp and the radix tile, group counts on both sides of one / two radix passes and of the device
path's capacity (above it the host sort runs: `partition_device` in ek_stats says which path ran), special and
badly-hashing keys, keys that are a prefix of a larger allocation (sentinels past n must never show up), an 8-byte but not
16-byte aligned input, repeated calls between evaluator work, and the Python enoki_b200.partition().

Key tables are drawn with rng.integers, never from a materialised value range (see test_partition in
test_gpu_zz_round2.py for why)."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CAPACITY = 1 << 16              # distinct values the device path groups
TILE = 4096                     # radix tile of ek_partition.cu
SENTINEL = np.uint64(0x5EA7_0000_DEAD_BEE0)
GUARD = 64

_libc = ctypes.CDLL(None)
_libc.free.argtypes = [ctypes.c_void_p]


def table(rng, k):
    cand = np.unique(rng.integers(1, 1 << 40, size=2 * k + 16, dtype=np.uint64))
    assert len(cand) >= k
    return rng.permutation(cand)[:k] * np.uint64(16)


def run(ek, keys, offset=0):
    """ek_partition over `keys` placed `offset` elements into a device buffer with GUARD sentinels after them.
    Returns (unique, counts, concatenated index lists, ran on the device)."""
    L = ek.lib()
    keys = np.ascontiguousarray(keys, np.uint64)
    n = len(keys)
    assert not (keys == SENTINEL).any()
    buf = np.full(offset + n + GUARD, SENTINEL, np.uint64)
    buf[offset:offset + n] = keys
    arr = ek.UInt64.copy(buf)
    base = arr.data() + offset * 8
    before = int(ek.stats().partition_device)
    uniq, counts, lists = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    assert L.ek_partition(n, base, ctypes.byref(uniq), ctypes.byref(counts), ctypes.byref(lists)) == 0, L.ek_last_error()
    device = int(ek.stats().partition_device) - before
    assert device in (0, 1)
    k = ctypes.cast(counts, ctypes.POINTER(ctypes.c_uint32))[0]
    cnt = np.ctypeslib.as_array(ctypes.cast(counts, ctypes.POINTER(ctypes.c_uint32)), shape=(k + 1,))[1:].copy()
    un = np.ctypeslib.as_array(ctypes.cast(uniq, ctypes.POINTER(ctypes.c_uint64)), shape=(k,)).copy()
    ptrs = np.ctypeslib.as_array(ctypes.cast(lists, ctypes.POINTER(ctypes.c_uint64)), shape=(k,)).copy()
    assert int(cnt.sum()) == n
    idx = np.empty(n, np.uint32)
    off = 0
    for p, c in zip(ptrs, cnt):
        L.ek_memcpy_from_device(idx[off:].ctypes.data, int(p), int(c) * 4)
        off += int(c)
    for p in ptrs:
        L.ek_free(int(p))
    L.ek_host_free(uniq)
    L.ek_host_free(counts)
    _libc.free(lists)
    del arr
    return un, cnt, idx, bool(device)


def check(ek, keys, device=True, offset=0):
    keys = np.asarray(keys, np.uint64)
    un, cnt, idx, on_device = run(ek, keys, offset)
    assert on_device == device, f"expected the {'device' if device else 'host'} path"
    want_u, want_c = np.unique(keys, return_counts=True)
    assert len(un) == len(want_u)
    assert (un == want_u).all() and (cnt == want_c).all()
    assert (idx == np.argsort(keys, kind="stable")).all()
    return un, cnt, idx


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, TILE - 1, TILE, TILE + 1, (1 << 20) + 3, 1 << 24])
def test_partition_sizes(gpu, n):
    rng = np.random.default_rng(n)
    k = min(n, 7)
    t = table(rng, k)
    check(gpu, t[rng.integers(0, k, n)] if n > k else t[:n])


@pytest.mark.parametrize("coherent", [False, True], ids=["random", "runs"])
@pytest.mark.parametrize("k", [1, 2, 255, 256, 257, 4096, CAPACITY - 1, CAPACITY])
def test_partition_groups(gpu, k, coherent):
    rng = np.random.default_rng(k * 2 + coherent)
    n = max(4 * k, 300_001)
    t = table(rng, k)
    if coherent:
        keys = t[(np.arange(n, dtype=np.int64) * k) // n]
    else:
        keys = t[rng.permutation(np.arange(n) % k)]         # every value present
    check(gpu, keys)


def test_partition_above_capacity_falls_back(gpu):
    rng = np.random.default_rng(77)
    k = CAPACITY + 1
    t = table(rng, k)
    check(gpu, t[rng.permutation(np.arange(3 * k) % k)], device=False)


def test_partition_special_keys(gpu):
    """0, 1, 2^63 - 1, 2^63, ~0, keys that differ only in the high 32 bits, multiples of 2^20 (hash quality)."""
    rng = np.random.default_rng(3)
    special = np.array([0, 1, (1 << 63) - 1, 1 << 63, (1 << 64) - 1, 5 << 32, 6 << 32, 1 << 20, 2 << 20], np.uint64)
    check(gpu, special[rng.integers(0, len(special), 500_000)])
    check(gpu, np.repeat(special, 50_000))
    high = (np.arange(1, 3001, dtype=np.uint64) << np.uint64(32)) | np.uint64(0x1000)
    check(gpu, high[rng.integers(0, len(high), 400_000)])
    mult = np.arange(1, 40_001, dtype=np.uint64) << np.uint64(20)
    check(gpu, mult[rng.integers(0, len(mult), 1_000_000)])


@pytest.mark.parametrize("value", [0, (1 << 64) - 1, 0x7F00_1234_5670])
def test_partition_single_value(gpu, value):
    check(gpu, np.full(1_000_003, value, np.uint64))


def test_partition_alternating(gpu):
    n = 1_000_001
    check(gpu, np.where(np.arange(n) % 2 == 0, np.uint64(0x1000), np.uint64(0x2000)))
    check(gpu, np.array([0x30, 0x10, 0x20], np.uint64)[np.arange(n) % 3])


def test_partition_misaligned_input(gpu):
    """Keys 8-byte but not 16-byte aligned."""
    rng = np.random.default_rng(8)
    for k, n in [(5, 100_001), (300, 200_003)]:
        t = table(rng, k)
        check(gpu, t[rng.integers(0, k, n)], offset=1)


def test_partition_repeated_with_evaluator_work(gpu):
    """Many calls in a row, between evaluator sweeps, give the same groups; after ek_malloc_trim the device memory is
    back where it was (every scratch buffer and output was released)."""
    ek = gpu
    L = ek.lib()
    rng = np.random.default_rng(21)
    n = 1 << 23
    t = table(rng, 300)
    keys = t[rng.integers(0, 300, n)]
    ek.cuda_sync(); L.ek_malloc_trim()
    free0, total = ctypes.c_size_t(), ctypes.c_size_t()
    L.ek_mem_get_info(ctypes.byref(free0), ctypes.byref(total))
    first = check(ek, keys)
    x = ek.Float32.copy(rng.uniform(-1, 1, 1 << 20).astype(np.float32))
    for i in range(6):
        y = ek.sin(x * float(i + 1)) + x
        s = float(ek.hsum(y).coeff(0))
        assert np.isfinite(s)
        again = check(ek, keys)
        assert all((a == b).all() for a, b in zip(first, again))
    del x, y
    ek.cuda_sync(); L.ek_malloc_trim()
    free1 = ctypes.c_size_t()
    L.ek_mem_get_info(ctypes.byref(free1), ctypes.byref(total))
    assert abs(free0.value - free1.value) < 16 << 20, (free0.value, free1.value)


def test_python_partition(gpu):
    ek = gpu
    rng = np.random.default_rng(4)
    t = table(rng, 600)
    keys = t[rng.integers(0, 600, 250_000)]
    groups = ek.partition(ek.UInt64.copy(keys))
    want_u, want_c = np.unique(keys, return_counts=True)
    assert [g[0] for g in groups] == [int(v) for v in want_u]
    assert [len(g[1]) for g in groups] == [int(c) for c in want_c]
    got = np.concatenate([g[1].numpy() for g in groups])
    assert (got == np.argsort(keys, kind="stable")).all()
    with pytest.raises(TypeError):
        ek.partition(ek.UInt32.copy(np.arange(4, dtype=np.uint32)))
