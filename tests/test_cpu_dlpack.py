"""CPU suite: DLPack export / import (enoki_b200/dlpack.py, ek_dlpack_export / ek_dlpack_import).  Everything here runs
without a device: arrays are mapped over fake device addresses (never dereferenced), and every check of an import is
made before any CUDA call."""
import ctypes
import gc
import threading

import pytest

F = 0x7f0000000000       # fake device address


@pytest.fixture()
def dl(ek):
    from enoki_b200 import dlpack
    gc.collect(); ek.lib().ek_sync()
    yield dlpack
    gc.collect(); ek.lib().ek_sync()


def test_struct_layouts_match_the_specification(dl):
    """sizes and offsets of dlpack.h's structures (ABI 1.0) on a 64-bit platform"""
    S, O = ctypes.sizeof, lambda cls, f: getattr(cls, f).offset
    assert S(dl.DLDevice) == 8 and O(dl.DLDevice, "device_id") == 4
    assert S(dl.DLDataType) == 4 and (O(dl.DLDataType, "bits"), O(dl.DLDataType, "lanes")) == (1, 2)
    assert S(dl.DLTensor) == 48
    assert [O(dl.DLTensor, f) for f in ("data", "device", "ndim", "dtype", "shape", "strides", "byte_offset")] == \
        [0, 8, 16, 20, 24, 32, 40]
    assert S(dl.DLManagedTensor) == 64
    assert [O(dl.DLManagedTensor, f) for f in ("dl_tensor", "manager_ctx", "deleter")] == [0, 48, 56]
    assert S(dl.DLPackVersion) == 8
    assert S(dl.DLManagedTensorVersioned) == 80
    assert [O(dl.DLManagedTensorVersioned, f) for f in ("version", "manager_ctx", "deleter", "flags", "dl_tensor")] == \
        [0, 8, 16, 24, 32]
    assert (dl.kDLCPU, dl.kDLCUDA) == (1, 2)
    assert (dl.kDLInt, dl.kDLUInt, dl.kDLFloat, dl.kDLBfloat, dl.kDLComplex, dl.kDLBool) == (0, 1, 2, 4, 5, 6)


TABLE = [("Float16", 2, 16), ("Float32", 2, 32), ("Float64", 2, 64), ("Int8", 0, 8), ("Int16", 0, 16), ("Int32", 0, 32),
         ("Int64", 0, 64), ("UInt8", 1, 8), ("UInt16", 1, 16), ("UInt32", 1, 32), ("UInt64", 1, 64), ("Mask", 6, 8)]


@pytest.mark.parametrize("versioned", [0, 1])
def test_dtype_table_round_trips(ek, dl, versioned):
    L = ek.lib()
    for k, (name, code, bits) in enumerate(TABLE):
        cls = getattr(ek, name)
        a = cls.map(F + 0x1000000 * k, 37)
        p = L.ek_dlpack_export(a.index, versioned, None)
        assert p, L.ek_last_error()
        m = ctypes.cast(p, ctypes.POINTER(dl.DLManagedTensorVersioned if versioned else dl.DLManagedTensor)).contents
        t = m.dl_tensor
        assert (t.dtype.code, t.dtype.bits, t.dtype.lanes) == (code, bits, 1), name
        assert t.data == F + 0x1000000 * k and (t.device.device_type, t.device.device_id) == (dl.kDLCUDA, L.ek_device())
        assert t.ndim == 1 and t.shape[0] == 37 and not t.strides and t.byte_offset == 0
        if versioned:
            assert (m.version.major, m.version.minor, m.flags) == (1, 0, 0)
        h = L.ek_dlpack_import(p, versioned)
        assert h, L.ek_last_error()
        b = ek.CUDAArray.from_index(h)
        assert L.ek_var_type(h) == cls.Type and L.ek_var_ptr(h) == F + 0x1000000 * k and L.ek_var_size(h) == 37
        del a, b
        L.ek_sync()


def test_pointer_arrays_are_not_exported(ek, dl):
    L = ek.lib()
    p = L.ek_var_register_ptr(F)
    assert not L.ek_dlpack_export(p, 1, None)
    assert b"ptr cannot be exported" in L.ek_last_error()
    L.ek_dec_ref_ext(p)


class Tensor:
    """a hand-built managed tensor with a counting deleter"""

    def __init__(self, dl, shape, code=2, bits=32, lanes=1, device=(2, None), strides=None, data=F, offset=0,
                 versioned=True, flags=0, major=1):
        import enoki_b200
        self.deleted = 0
        M = dl.DLManagedTensorVersioned if versioned else dl.DLManagedTensor
        self.m = M()
        self.shape = (ctypes.c_int64 * max(len(shape), 1))(*shape)
        self.strides = (ctypes.c_int64 * len(strides))(*strides) if strides is not None else None
        t = self.m.dl_tensor
        t.data = data
        t.device.device_type = device[0]
        t.device.device_id = enoki_b200.lib().ek_device() if device[1] is None else device[1]
        t.ndim = len(shape)
        t.dtype.code, t.dtype.bits, t.dtype.lanes = code, bits, lanes
        t.shape = self.shape
        t.strides = self.strides
        t.byte_offset = offset
        if versioned:
            self.m.version.major, self.m.version.minor, self.m.flags = major, 0, flags
        self.versioned = versioned
        self._fn = dict(M._fields_)["deleter"](self._delete)
        self.m.deleter = self._fn

    def _delete(self, ptr):
        self.deleted += 1

    @property
    def ptr(self):
        return ctypes.addressof(self.m)

    def __dlpack__(self, stream=None, max_version=None):
        from enoki_b200 import dlpack
        # (with the destructor the protocol prescribes, which this package's capsules use as well)
        return dlpack._capsule_new(self.ptr, dlpack.VERSIONED if self.versioned else dlpack.LEGACY, dlpack._DESTRUCTOR)


@pytest.mark.parametrize("case, message", [
    (dict(shape=[8], device=(1, 0)), "device type 1 is not supported"),
    (dict(shape=[8], device=(2, 1)), "the tensor is on CUDA device 1, the backend runs on device 0"),
    (dict(shape=[8], lanes=4), "4 lanes is not supported"),
    (dict(shape=[8], code=4, bits=16), "dtype bfloat16 is not supported"),
    (dict(shape=[8], code=5, bits=64), "dtype complex64 is not supported"),
    (dict(shape=[8], code=10, bits=8), "dtype float8 (type code 10) is not supported"),
    (dict(shape=[8], code=2, bits=8), "dtype float8 is not supported"),
    (dict(shape=[8], code=6, bits=16), "dtype bool16 is not supported"),
    (dict(shape=[4, 6], strides=[1, 4]), "strides are not C-contiguous (dimension 1 has stride 4"),
    (dict(shape=[4, 6], strides=[12, 2]), "strides are not C-contiguous"),
    (dict(shape=[1 << 16, (1 << 16) + 1]), "size: arrays with more than 2^32-1 entries are not supported"),
    (dict(shape=[1 << 32]), "more than 2^32-1 entries"),
    (dict(shape=[3, 0]), "size zero"),
    (dict(shape=[8], offset=2), "not aligned to its 4-byte elements"),
    (dict(shape=[8], data=0), "null data pointer"),
    (dict(shape=[8], flags=1), "read-only tensors are not supported"),
    (dict(shape=[8], major=2), "DLPack version 2.0 is not supported"),
])
def test_import_refusals_name_the_reason(ek, dl, case, message):
    if "device 1" in message and ek.lib().ek_device() != 0:
        pytest.skip("the backend does not run on device 0 here")
    t = Tensor(dl, **case)
    L = ek.lib()
    assert L.ek_dlpack_import(t.ptr, 1) == 0
    assert message in L.ek_last_error().decode()
    # refused: the tensor is still the caller's, and nothing called its deleter
    L.ek_sync()
    assert t.deleted == 0
    # the Python path raises, and the capsule (unconsumed) releases the tensor when it goes
    with pytest.raises(ek.EnokiError, match="ek_dlpack_import"):
        ek.from_dlpack(t)
    gc.collect()
    assert t.deleted == 1


def test_import_accepts_any_c_contiguous_layout(ek, dl):
    L = ek.lib()
    for case, n in ((dict(shape=[4, 6], strides=[6, 1]), 24), (dict(shape=[4, 1, 6], strides=[6, 99, 1]), 24),
                    (dict(shape=[]), 1), (dict(shape=[2, 3, 5], offset=4), 30), (dict(shape=[7], versioned=False), 7)):
        t = Tensor(dl, **case)
        h = L.ek_dlpack_import(t.ptr, int(t.versioned))
        assert h, L.ek_last_error()
        assert L.ek_var_size(h) == n and L.ek_var_ptr(h) == F + case.get("offset", 0)
        L.ek_dec_ref_ext(h)
        assert t.deleted == 0                   # ... until the next entry
        L.ek_sync()
        assert t.deleted == 1


def test_freed_import_calls_the_deleter_once_and_never_reaches_the_allocator(ek, dl):
    L = ek.lib()
    t = Tensor(dl, shape=[256])
    a = ek.from_dlpack(t)
    assert type(a) is ek.Float32 and L.ek_var_ptr(a.index) == F
    b = a * 2.0                                 # a recorded use keeps the variable alive
    del a
    L.ek_sync()
    assert t.deleted == 0
    del b
    assert t.deleted == 0
    L.ek_sync()
    assert t.deleted == 1
    L.ek_malloc_trim()                          # (would hand the fake address to cudaFree if it were on a free list)
    L.ek_sync()
    assert t.deleted == 1


def test_capsule_names_and_consumption(ek, dl):
    a = ek.Float32.map(F, 16)
    valid = lambda cap, name: bool(dl._capsule_valid(ctypes.c_void_p(id(cap)), name))
    assert valid(a.__dlpack__(stream=-1), dl.LEGACY)
    assert valid(a.__dlpack__(stream=-1, max_version=(0, 8)), dl.LEGACY)
    assert valid(a.__dlpack__(stream=-1, max_version=(1, 0)), dl.VERSIONED)
    assert valid(a.__dlpack__(stream=-1, max_version=(1, 3)), dl.VERSIONED)
    assert a.__dlpack_device__() == (dl.kDLCUDA, ek.lib().ek_device())
    with pytest.raises(BufferError, match="use .torch"):
        a.__dlpack__(stream=-1, copy=True)
    with pytest.raises(BufferError):
        a.__dlpack__(stream=-1, dl_device=(dl.kDLCPU, 0))
    with pytest.raises(ValueError, match="stream 0"):
        a.__dlpack__(stream=0)

    # a consumer renames the capsule it takes over; the destructor leaves a consumed capsule alone
    t = Tensor(dl, shape=[16])
    cap = t.__dlpack__()

    class Producer:
        def __dlpack__(self, stream=None, max_version=None):
            return cap
    b = ek.from_dlpack(Producer())
    assert valid(cap, dl.USED_VERSIONED) and not valid(cap, dl.VERSIONED)
    del cap
    gc.collect()
    assert t.deleted == 0
    del b
    ek.lib().ek_sync()
    assert t.deleted == 1

    # a legacy producer (no max_version) gives a "dltensor" capsule, renamed "used_dltensor"
    t2 = Tensor(dl, shape=[16], versioned=False)
    seen = []

    class Legacy:
        def __dlpack__(self, stream=None):
            seen.append(t2.__dlpack__())
            return seen[-1]
    c = ek.Float32.from_dlpack(Legacy())
    assert valid(seen[0], dl.USED_LEGACY)
    with pytest.raises(TypeError, match="holds Float32"):
        ek.Int32.from_dlpack(Tensor(dl, shape=[4]))
    del c, seen
    ek.lib().ek_sync()
    assert t2.deleted == 1


def test_unconsumed_export_capsule_releases_its_reference(ek, dl):
    L = ek.lib()
    a = ek.Float32.map(F, 16)
    h = a.index
    cap = a.__dlpack__(stream=-1, max_version=(1, 0))
    del a
    assert L.ek_var_size(h) == 16               # held by the capsule
    del cap                                     # the destructor runs the deleter: the release is queued ...
    assert L.ek_var_size(h) == 16
    L.ek_sync()                                 # ... and done at the next entry
    assert L.ek_var_size(h) == 0


def test_export_dropped_on_another_thread_is_released_on_the_owning_thread(ek, dl):
    L = ek.lib()
    a = ek.Float32.map(F, 16)
    h = a.index
    box = [a.__dlpack__(stream=-1)]
    del a
    th = threading.Thread(target=box.clear)
    th.start(); th.join()
    assert not box and L.ek_var_size(h) == 16   # the deleter made no runtime call on that thread
    L.ek_eval()                                 # the next entry on this thread releases it
    assert L.ek_var_size(h) == 0
