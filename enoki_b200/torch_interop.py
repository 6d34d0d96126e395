"""PyTorch interop (SURVEY 8f row 2; reference: src/python/common.h:1085-1215 `enoki_to_torch` / `torch_to_enoki`,
tests/python/test_pytorch.py:6-29).  Both directions copy device-to-device, as the reference does: an Enoki array and a
torch tensor never alias, so neither allocator has to know about the other.  Ordering between torch's current stream
and the backend's stream is made explicit (synchronise the producer before the copy, the backend's stream after it)."""
import numpy as np

from . import (CUDAArray, Float32, Float64, Int32, UInt32, Int64, UInt64, Mask, lib,
               EK_FLOAT16, EK_FLOAT32, EK_FLOAT64, EK_INT32, EK_UINT32, EK_INT64, EK_UINT64, EK_BOOL)


def _torch():
    import torch
    return torch


def _dtype_of(cls):
    t = _torch()
    return {EK_FLOAT16: t.float16, EK_FLOAT32: t.float32, EK_FLOAT64: t.float64, EK_INT32: t.int32, EK_UINT32: t.int32,
            EK_INT64: t.int64, EK_UINT64: t.int64, EK_BOOL: t.bool}[cls.Type]


def to_torch(a):
    """Enoki array -> new torch tensor on the same device (unsigned integers arrive as the signed dtype of the same
    width, like the reference's numpy/torch casters)."""
    t = _torch()
    n = a.size()
    a.eval()
    out = t.empty(n, dtype=_dtype_of(type(a)), device=f"cuda:{t.cuda.current_device()}")
    if n:
        t.cuda.current_stream().synchronize()           # the fresh tensor's memory may still be in use on torch's stream
        lib().ek_memcpy_device_async(out.data_ptr(), lib().ek_var_ptr(a.index), n * out.element_size())
        lib().ek_sync()
    return out


def from_torch(cls, tensor):
    """torch CUDA tensor -> new Enoki array of class `cls` (contiguous copy)."""
    t = _torch()
    want = _dtype_of(cls)
    x = tensor.detach()
    if x.dtype != want:
        x = x.to(want)
    x = x.contiguous().reshape(-1)
    if not x.is_cuda:
        return cls(x.numpy())
    n = x.numel()
    if n == 0:
        raise ValueError("from_torch(): empty tensor")
    r = cls.empty(n)
    t.cuda.current_stream().synchronize()               # the tensor's producer has to be done before our stream reads it
    lib().ek_memcpy_device_async(lib().ek_var_ptr(r.index), x.data_ptr(), n * x.element_size())
    lib().ek_sync()                                      # ... and x may be freed by torch as soon as we return
    return r


def _install():
    CUDAArray.torch = to_torch
    CUDAArray.from_torch = classmethod(from_torch)
    from .autodiff import FloatD
    FloatD.torch = lambda self: to_torch(self.value)
    FloatD.from_torch = staticmethod(lambda tensor: FloatD(from_torch(Float32, tensor)))


_install()
