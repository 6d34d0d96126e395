"""Zero-copy exchange of device arrays with torch, CuPy, JAX and anything else that speaks DLPack.

    t = torch.from_dlpack(a)        # a torch tensor aliasing the Enoki array `a`
    b = enoki_b200.from_dlpack(t)   # an Enoki array aliasing the torch tensor `t`

This is the aliasing path: both sides see one buffer, writes on either side are seen by the other, and nothing is
copied.  `.torch()` / `from_torch()` (torch_interop.py) are the copying path: use them for an independent copy, or to
map unsigned arrays to torch's signed dtypes.

Ordering follows the array API's `__dlpack__` protocol and needs no host synchronisation:
- export: the consumer passes its stream; it waits (on the device) for the backend's work on the array.  When the
  consumer drops the tensor, the release is ordered after the work the consumer had enqueued on that stream by then.
- import: `from_dlpack` passes the backend's stream to the producer, which makes it wait for the producer's work.  The
  producer's buffer is handed back (its deleter is called) once the backend's last use of it has completed.
A consumer may drop an exported tensor on any thread: the release is queued and done on the thread that owns the
backend, at its next call into it (include/enoki_b200.h, ek_dlpack_export).
"""
import ctypes

from . import CUDAArray, _BY_TYPE, _check, lib

kDLCPU, kDLCUDA = 1, 2
kDLInt, kDLUInt, kDLFloat, kDLOpaqueHandle, kDLBfloat, kDLComplex, kDLBool = range(7)


# ---- the structures of include/enoki_b200_dlpack.h ------------------------------------------------
class DLDevice(ctypes.Structure):
    _fields_ = [("device_type", ctypes.c_int32), ("device_id", ctypes.c_int32)]


class DLDataType(ctypes.Structure):
    _fields_ = [("code", ctypes.c_uint8), ("bits", ctypes.c_uint8), ("lanes", ctypes.c_uint16)]


class DLTensor(ctypes.Structure):
    _fields_ = [("data", ctypes.c_void_p), ("device", DLDevice), ("ndim", ctypes.c_int32), ("dtype", DLDataType),
                ("shape", ctypes.POINTER(ctypes.c_int64)), ("strides", ctypes.POINTER(ctypes.c_int64)),
                ("byte_offset", ctypes.c_uint64)]


class DLManagedTensor(ctypes.Structure):
    pass


DLManagedTensor._fields_ = [("dl_tensor", DLTensor), ("manager_ctx", ctypes.c_void_p),
                            ("deleter", ctypes.CFUNCTYPE(None, ctypes.POINTER(DLManagedTensor)))]


class DLPackVersion(ctypes.Structure):
    _fields_ = [("major", ctypes.c_uint32), ("minor", ctypes.c_uint32)]


class DLManagedTensorVersioned(ctypes.Structure):
    pass


DLManagedTensorVersioned._fields_ = [("version", DLPackVersion), ("manager_ctx", ctypes.c_void_p),
                                     ("deleter", ctypes.CFUNCTYPE(None, ctypes.POINTER(DLManagedTensorVersioned))),
                                     ("flags", ctypes.c_uint64), ("dl_tensor", DLTensor)]


# ---- capsules (the names must outlive the capsules that point at them: module constants) -----------
LEGACY, VERSIONED = b"dltensor", b"dltensor_versioned"
USED_LEGACY, USED_VERSIONED = b"used_dltensor", b"used_dltensor_versioned"

_api = ctypes.pythonapi
_capsule_new = ctypes.PYFUNCTYPE(ctypes.py_object, ctypes.c_void_p, ctypes.c_char_p, ctypes.c_void_p)(("PyCapsule_New", _api))
_capsule_valid = ctypes.PYFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_char_p)(("PyCapsule_IsValid", _api))
_capsule_pointer = ctypes.PYFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p, ctypes.c_char_p)(("PyCapsule_GetPointer", _api))
_capsule_set_name = ctypes.PYFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_char_p)(("PyCapsule_SetName", _api))


def _release(managed, versioned):
    """call a managed tensor's deleter"""
    ptr = ctypes.cast(managed, ctypes.POINTER(DLManagedTensorVersioned if versioned else DLManagedTensor))
    if ptr.contents.deleter:
        ptr.contents.deleter(ptr)


@ctypes.CFUNCTYPE(None, ctypes.c_void_p)
def _capsule_destructor(capsule):
    # a consumer renames the capsule when it takes the tensor over; one that was never consumed still owns it
    for name, versioned in ((VERSIONED, True), (LEGACY, False)):
        if _capsule_valid(capsule, name):
            _release(_capsule_pointer(capsule, name), versioned)


_DESTRUCTOR = ctypes.cast(_capsule_destructor, ctypes.c_void_p)


# ---- the protocol ----------------------------------------------------------------------------------
def _dlpack_device(self):
    """(kDLCUDA, device): where __dlpack__ exports the array"""
    return (kDLCUDA, lib().ek_device())


def _dlpack(self, stream=None, max_version=None, dl_device=None, copy=None):
    """Export the array as a DLPack capsule that aliases its buffer (array API protocol).

    stream: the consumer's CUDA stream as an integer; it is made to wait for the backend's work on the array.  None
    means the legacy default stream (1), 2 the per-thread default stream, -1 no ordering at all.  max_version >= (1, 0)
    gives the versioned capsule "dltensor_versioned", anything else the legacy "dltensor".  copy=True is refused: use
    .torch() for an independent copy."""
    if copy:
        raise BufferError("__dlpack__(copy=True): a DLPack export aliases the array; use .torch() for a copy")
    if dl_device is not None and tuple(dl_device) != self.__dlpack_device__():
        raise BufferError(f"__dlpack__(): the array is on {self.__dlpack_device__()}, not on {tuple(dl_device)}")
    if stream is None:
        stream = 1
    if stream == 0:
        raise ValueError("__dlpack__(): stream 0 is ambiguous for CUDA; pass 1 for the legacy default stream")
    versioned = max_version is not None and tuple(max_version) >= (1, 0)
    if stream != -1:
        self.eval()
        _check(0, lib().ek_stream_signal_external(stream) == 0)
    p = lib().ek_dlpack_export(self.index, int(versioned), None if stream == -1 else stream)
    _check(p, bool(p))
    return _capsule_new(p, VERSIONED if versioned else LEGACY, _DESTRUCTOR)


def from_dlpack(obj, cls=None):
    """Import `obj` (a torch tensor, CuPy / JAX array, ... with `__dlpack__`) as an array that aliases its buffer.

    The array class follows the dtype (a bool tensor gives a Mask); with `cls` the dtype must be that class's.  Only
    C-contiguous CUDA memory on the backend's device is accepted: call .contiguous() on a strided view first.  The
    producer's work on the buffer is ordered before the backend's without a host synchronisation.  Use from_torch()
    instead for an independent copy."""
    if not hasattr(obj, "__dlpack__"):
        raise TypeError(f"from_dlpack(): {type(obj).__name__} does not implement __dlpack__")
    # (with no device the backend has no stream, and no work to order: the import is still checked)
    stream = lib().ek_stream() or -1
    try:
        capsule = obj.__dlpack__(stream=stream, max_version=(1, 0))
    except TypeError:                       # a producer of the legacy protocol
        capsule = obj.__dlpack__(stream=stream)
    cap = ctypes.c_void_p(id(capsule))
    versioned = bool(_capsule_valid(cap, VERSIONED))
    if not versioned and not _capsule_valid(cap, LEGACY):
        raise BufferError("from_dlpack(): __dlpack__ did not return an unconsumed DLPack capsule")
    h = lib().ek_dlpack_import(_capsule_pointer(cap, VERSIONED if versioned else LEGACY), int(versioned))
    _check(h, h != 0)                       # refused: the capsule still owns the tensor
    _capsule_set_name(cap, USED_VERSIONED if versioned else USED_LEGACY)
    r = _BY_TYPE[lib().ek_var_type(h)].from_index(h)
    if cls is not None and cls is not CUDAArray and type(r) is not cls:
        raise TypeError(f"{cls.__name__}.from_dlpack(): the tensor holds {type(r).__name__} elements")
    return r


def _install():
    CUDAArray.__dlpack__ = _dlpack
    CUDAArray.__dlpack_device__ = _dlpack_device
    CUDAArray.from_dlpack = classmethod(lambda cls, obj: from_dlpack(obj, cls))
    from .autodiff import FloatD       # the detached value only: gradients do not cross by alias
    FloatD.__dlpack__ = lambda self, *a, **kw: self.value.__dlpack__(*a, **kw)
    FloatD.__dlpack_device__ = lambda self: self.value.__dlpack_device__()


_install()
