"""GPU: sharing device arrays with torch through DLPack, without copies (enoki_b200/dlpack.py).  Aliasing for every type
and size class, imports feeding both sweep kernels (misaligned views among them), writes seen across, stream ordering
with no host synchronisation, lifetimes and deleters, the torch.autograd.Function bridge, and tests/cpp/dlpack_check."""
import gc
import os
import subprocess
import threading

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

TYPES = [("Float16", torch.float16, np.float16), ("Float32", torch.float32, np.float32),
         ("Float64", torch.float64, np.float64), ("Int8", torch.int8, np.int8), ("UInt8", torch.uint8, np.uint8),
         ("Int16", torch.int16, np.int16), ("UInt16", torch.uint16, np.uint16), ("Int32", torch.int32, np.int32),
         ("UInt32", torch.uint32, np.uint32), ("Int64", torch.int64, np.int64), ("UInt64", torch.uint64, np.uint64),
         ("Mask", torch.bool, np.bool_)]
SLEEP = 1 << 30          # torch.cuda._sleep cycles: about half a second on an H100


@pytest.fixture(autouse=True)
def clean(ek, gpu):
    gc.collect(); ek.lib().ek_sync()
    yield
    ek.lib().ek_set_fast_mode(1)
    gc.collect(); ek.lib().ek_sync()


def _data(npt, n, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, n * np.dtype(npt).itemsize, dtype=np.uint8).view(npt) if npt is not np.bool_ \
        else rng.integers(0, 2, n).astype(np.bool_)


def _bytes(t):
    return t.detach().view(torch.uint8).cpu().numpy().tobytes()


@pytest.mark.parametrize("n", [1, 31, 4097, (1 << 20) + 3])
def test_both_directions_alias_every_type(ek, n):
    L = ek.lib()
    for k, (name, tdt, npt) in enumerate(TYPES):
        cls = getattr(ek, name)
        host = _data(npt, n, k)
        a = cls.copy(host)
        t = torch.from_dlpack(a)
        assert t.dtype == tdt and t.shape == (n,) and t.is_cuda
        assert t.data_ptr() == L.ek_var_ptr(a.index), name
        assert _bytes(t) == host.tobytes(), name
        b = ek.from_dlpack(t)
        assert type(b) is cls and L.ek_var_ptr(b.index) == t.data_ptr()
        u = torch.from_numpy(host.view(np.uint8).copy()).cuda().view(tdt)      # a tensor torch allocated
        c = ek.from_dlpack(u)
        assert type(c) is cls and L.ek_var_ptr(c.index) == u.data_ptr()
        assert c.numpy().tobytes() == host.tobytes(), name
        del a, t, b, u, c


C2 = lambda ek, x: (lambda t: ek.fmadd(ek.sin(ek.fmadd(x[3], ek.exp(-(t * t)), x[0])), x[1], ek.sqrt(abs(t))))(
    ek.fmadd(x[0], x[1], x[2]))


@pytest.mark.parametrize("fast", [1, 0])
def test_imports_feed_both_sweep_kernels(ek, fast):
    """C2 over imported tensors (one of them a view t[1:] that starts 4 bytes into its buffer) equals C2 over copies"""
    L = ek.lib()
    L.ek_set_fast_mode(fast)
    n = (1 << 20) + 77
    g = torch.Generator(device="cuda").manual_seed(5)
    ts = [torch.rand(n + (k == 2), device="cuda", generator=g) * 8 - 4 for k in range(4)]
    views = [ts[0], ts[1], ts[2][1:], ts[3]]
    assert views[2].data_ptr() % 16 == 4
    xs = [ek.from_dlpack(v) for v in views]
    assert L.ek_var_ptr(xs[2].index) == views[2].data_ptr()
    L.ek_stats_reset()
    got = C2(ek, xs).numpy()
    assert (ek.stats().fast_launches > 0) == bool(fast)
    want = C2(ek, [ek.Float32.copy(v.cpu().numpy()) for v in views]).numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_writes_are_seen_in_both_directions(ek):
    L = ek.lib()
    n = 10_007
    # torch writes into an exported buffer; a later evaluation reads them
    a = ek.Float32.copy(np.arange(n, dtype=np.float32))
    t = torch.from_dlpack(a)
    t.mul_(3)
    L.ek_stream_wait_external(torch.cuda.current_stream().cuda_stream)
    assert np.array_equal((a + 1.0).numpy(), np.arange(n, dtype=np.float32) * 3 + 1)
    # an Enoki scatter into an imported buffer; torch reads it
    u = torch.zeros(n, dtype=torch.int32, device="cuda")
    b = ek.from_dlpack(u)
    idx = ek.UInt32.arange(n // 2) * 2
    ek.scatter(b, ek.Int32(idx) + 7, idx)
    ek.cuda_eval()
    L.ek_stream_signal_external(torch.cuda.current_stream().cuda_stream)
    want = np.zeros(n, np.int32)
    want[0:n - 1:2] = np.arange(0, n - 1, 2) + 7
    assert np.array_equal(u.cpu().numpy(), want)
    del a, t, b, u


def test_import_waits_for_a_delayed_producer(ek):
    """the producer writes on a side stream after a long sleep; the import reads what it wrote (no host sync)"""
    n = 1 << 22
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        t = torch.zeros(n, device="cuda")
        torch.cuda._sleep(SLEEP)
        t.fill_(3.0)
        a = ek.from_dlpack(t)          # __dlpack__(stream=backend's) on the side stream
    out = (a * 2.0 + 1.0).numpy()
    assert (out == 7.0).all()
    del a, t


def test_consumer_on_a_side_stream_sees_a_finished_sweep(ek):
    n = 1 << 26
    x = ek.Float32.linspace(-3.0, 3.0, n)
    y = x
    for _ in range(48):
        y = ek.sin(y) * 0.75 + x
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        t = torch.from_dlpack(y)       # the side stream waits for the sweep
        copy = t.clone()
    side.synchronize()
    want = y.numpy()
    assert np.array_equal(copy.cpu().numpy().view(np.uint32), want.view(np.uint32))
    del x, y, t, copy


class Producer:
    """a DLPack producer around a torch tensor with a counting deleter: the tensor is dropped when the deleter runs"""

    def __init__(self, tensor):
        import ctypes
        from enoki_b200 import dlpack
        self.tensor, self.deleted = tensor, 0
        self.m = dlpack.DLManagedTensorVersioned()
        self.shape = (ctypes.c_int64 * 1)(tensor.numel())
        d = self.m.dl_tensor
        d.data, d.device.device_type, d.device.device_id = tensor.data_ptr(), dlpack.kDLCUDA, tensor.device.index
        d.ndim, d.shape, d.byte_offset = 1, self.shape, 0
        d.dtype.code, d.dtype.bits, d.dtype.lanes = dlpack.kDLFloat, 32, 1
        self.m.version.major = 1
        self.fn = dict(dlpack.DLManagedTensorVersioned._fields_)["deleter"](self._delete)
        self.m.deleter = self.fn

    def _delete(self, ptr):
        self.deleted += 1
        self.tensor = None

    def __dlpack__(self, stream=None, max_version=None):
        import ctypes
        from enoki_b200 import dlpack
        import enoki_b200
        enoki_b200.lib().ek_stream_wait_external(torch.cuda.current_stream().cuda_stream)
        return dlpack._capsule_new(ctypes.addressof(self.m), dlpack.VERSIONED, dlpack._DESTRUCTOR)


def test_producer_deleter_runs_once_after_the_last_use(ek):
    L = ek.lib()
    n = 1 << 24
    t = torch.full((n,), 2.0, device="cuda")
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP)
    L.ek_stream_wait_external(side.cuda_stream)        # the backend's stream is held up behind the sleep
    p = Producer(t)
    del t
    a = ek.from_dlpack(p)
    b = a * 3.0
    b.eval()
    held = torch.cuda.memory_allocated()
    del a                                              # the last reference: b is evaluated (enqueued, not run)
    ek.cuda_eval()                                     # an entry: the release is not due yet
    assert p.deleted == 0 and p.tensor is not None and torch.cuda.memory_allocated() == held
    ek.cuda_sync()                                     # waits for the last use, then calls the deleter
    assert p.deleted == 1 and p.tensor is None
    assert torch.cuda.memory_allocated() <= held - 4 * n
    assert (b.numpy() == 6.0).all()
    ek.cuda_sync()
    assert p.deleted == 1


def test_either_side_may_go_first(ek):
    n = 4099
    ref = np.arange(n, dtype=np.float32)
    a = ek.Float32.copy(ref)
    t = torch.from_dlpack(a)
    del a
    ek.cuda_sync()
    assert np.array_equal(t.cpu().numpy(), ref)
    u = torch.from_numpy(ref * 2).cuda()
    b = ek.from_dlpack(u)
    del u
    gc.collect()
    assert np.array_equal(b.numpy(), ref * 2)
    del t, b


def test_export_dropped_on_a_thread_is_released_on_the_main_thread(ek):
    L = ek.lib()
    n = 1 << 16
    a = ek.Float32.copy(np.ones(n, np.float32))
    h = a.index
    box = [torch.from_dlpack(a)]
    del a
    th = threading.Thread(target=box.clear)
    th.start(); th.join()
    assert not box
    assert L.ek_var_size(h) == n                       # nothing was released on that thread
    L.ek_eval()                                        # the next entry on the owning thread
    assert L.ek_var_size(h) == 0


def test_freed_import_never_reaches_the_allocator(ek):
    L = ek.lib()
    n = 1 << 20
    t = torch.arange(n, dtype=torch.float32, device="cuda")
    ptr = t.data_ptr()
    a = ek.from_dlpack(t)
    (a + 1.0).eval()
    del a
    ek.cuda_sync()
    blocks = [L.ek_malloc(4 * n) for _ in range(4)]
    assert ptr not in blocks
    for p in blocks:
        L.ek_free(p)
    L.ek_malloc_trim()
    assert t.sum().item() == n * (n - 1) / 2
    del t


def test_round_trip_aliases_and_frees_once(ek):
    L = ek.lib()
    n = 1 << 20
    a = ek.Float32.copy(np.full(n, 1.5, np.float32))
    ptr = L.ek_var_ptr(a.index)
    t = torch.from_dlpack(a)
    b = ek.from_dlpack(t)
    assert L.ek_var_ptr(b.index) == ptr and t.data_ptr() == ptr
    assert (b * 2.0).numpy()[0] == 3.0
    del a, t, b
    gc.collect()
    ek.cuda_sync()
    blocks = [L.ek_malloc(4 * n) for _ in range(3)]
    assert blocks.count(ptr) == 1                      # back on the free list, once
    for p in blocks:
        L.ek_free(p)


def _fn(ek, aliasing):
    import enoki_b200.torch_interop  # noqa: F401  (.torch() / from_torch())
    from enoki_b200 import autodiff as ad
    to_ek = (lambda x: ek.Float32.from_dlpack(x.detach().contiguous())) if aliasing else \
        (lambda x: ek.Float32.from_torch(x))
    to_torch = (lambda a: torch.from_dlpack(a)) if aliasing else (lambda a: a.torch())

    class EnokiFn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, y):
            ctx.in1 = ad.FloatD(to_ek(x)); ctx.in2 = ad.FloatD(to_ek(y))
            ad.set_requires_gradient(ctx.in1, x.requires_grad)
            ad.set_requires_gradient(ctx.in2, y.requires_grad)
            ctx.out = ctx.in1 * ad.sin(ctx.in2) + ad.exp(ctx.in1)
            out = to_torch(ctx.out.value)
            ek.lib().ek_malloc_trim()
            return out

        @staticmethod
        def backward(ctx, grad_out):
            ad.set_gradient(ctx.out, to_ek(grad_out))
            ad.backward_static()
            res = (to_torch(ad.gradient(ctx.in1)) if ctx.in1.requires_gradient() else None,
                   to_torch(ad.gradient(ctx.in2)) if ctx.in2.requires_gradient() else None)
            del ctx.out, ctx.in1, ctx.in2
            ek.lib().ek_malloc_trim()
            return res
    return EnokiFn


def test_autograd_bridge_by_alias_equals_the_copying_one(ek):
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(4096, device="cuda", generator=g, requires_grad=True)
    y = torch.randn(4096, device="cuda", generator=g, requires_grad=True)
    w = torch.randn(4096, device="cuda", generator=g)
    results = []
    for aliasing in (False, True):
        out = _fn(ek, aliasing).apply(x, y)
        (out * w).sum().backward()
        results.append((out.detach().clone(), x.grad.clone(), y.grad.clone()))
        x.grad = None; y.grad = None
        del out
    for c, a in zip(*results):
        assert torch.equal(c.view(torch.int32), a.view(torch.int32))


def test_cpp_dlpack_check(gpu):
    exe = os.path.join(HERE, "cpp", "dlpack_check")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/dlpack_check is built only where the reference headers exist")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert "dlpack_check ok" in r.stdout
