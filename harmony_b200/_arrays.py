"""Caller arrays at the library's boundary.  Nothing here loads the CUDA library, and torch is imported only where a
tensor was given or is made."""
import ctypes

import numpy as np

from .utils import is_cuda_tensor

DTYPE = {"float32": 0, "float64": 1}   # enum hb_dtype


def device_rows(obj, X, what):
    """An [n, d] float32 / float64 CUDA tensor on ``obj``'s device -> (the tensor to read, pointer, hb_dtype, row
    stride).  Rows with unit column stride are read in place, any other layout is made contiguous first."""
    import torch
    if X.dtype not in (torch.float32, torch.float64):
        raise TypeError(f"{what} must be float32 or float64, not {X.dtype}")
    if X.device.index != obj._scalar("device"):
        raise ValueError(f"{what} is on {X.device}, the harmony object on cuda:{obj._scalar('device')}")
    if X.shape[0] > 1 and not (X.stride(1) == 1 and X.stride(0) >= X.shape[1]):
        X = X.contiguous()
    ld = X.stride(0) if X.shape[0] > 1 else X.shape[1]
    return X, ctypes.c_void_p(X.data_ptr()), DTYPE[str(X.dtype)[6:]], int(ld)


def to_device(obj, a):
    """A host array -> a tensor on ``obj``'s device: float64 stays float64 (the library rounds after centring),
    anything else becomes float32."""
    import torch
    a = np.ascontiguousarray(a, dtype=np.float64 if a.dtype == np.float64 else np.float32)
    return torch.as_tensor(a).to(torch.device("cuda", obj._scalar("device")))


def current_stream(device):
    """The current torch stream of ``device``, which the library orders its call on."""
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def resolve_device(device, X, what):
    """The device a call on ``X`` runs on: a CUDA ``X``'s own, which ``device`` must match when given; else ``device``."""
    if not is_cuda_tensor(X):
        return device
    if device is not None and int(device) != X.device.index:
        raise ValueError(f"device={device} differs from the device of {what} ({X.device})")
    return X.device.index


def factorise(column, device=None):
    """A label column -> (sorted unique levels, int32 codes).  A CUDA column is factorised on its device; a host
    column gives numpy arrays, with the codes moved to ``device`` when it is given."""
    if is_cuda_tensor(column):
        import torch
        levels, codes = torch.unique(column, sorted=True, return_inverse=True)
        return levels, codes.to(torch.int32)
    levels, codes = np.unique(column, return_inverse=True)
    codes = codes.reshape(-1).astype(np.int32)
    if device is not None:
        import torch
        codes = torch.from_numpy(codes).to(device)
    return levels, codes
