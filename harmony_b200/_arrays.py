"""Caller arrays at the library's boundary.  Nothing here loads the CUDA library, and torch is imported only where a
tensor was given or is made."""
import ctypes

import numpy as np

from .utils import is_cuda_tensor

DTYPE = {"float32": 0, "float64": 1}   # enum hb_dtype
MAX_D = 128   # the widest embedding the scores (knn, LISI, silhouette) take


def embedding(X, what):
    """An embedding's rows: a CUDA tensor as it is, anything else as a numpy array; 2-D with 1 <= d <= MAX_D."""
    if not is_cuda_tensor(X):
        X = np.asarray(X)
    if X.ndim != 2:
        raise ValueError(f"{what} must be an [N, d] matrix")
    if not 1 <= X.shape[1] <= MAX_D:
        raise ValueError(f"d = {X.shape[1]} is not supported (1 <= d <= {MAX_D})")
    return X


def check_two_rows(X, what="X"):
    """The refusal of the scores that compare rows with each other: ``what`` needs at least 2 rows."""
    if X.shape[0] < 2:
        raise ValueError(f"{what} has {X.shape[0]} rows, at least 2 are needed")


def row_layout(t, width):
    """A 2-D tensor of rows of ``width`` elements -> (the tensor the library reads, its row stride ``ld``).  Rows with
    unit column stride and a row stride of at least ``width`` are read in place; any other layout is made contiguous
    first, a single row whose column stride is not 1 included."""
    if not (t.stride(1) == 1 and (t.shape[0] == 1 or t.stride(0) >= width)):
        t = t.contiguous()
    return t, int(t.stride(0) if t.shape[0] > 1 else width)


def device_rows(obj, X, what):
    """An [n, d] float32 / float64 CUDA tensor on ``obj``'s device -> (the tensor to read, pointer, hb_dtype, row
    stride), laid out by ``row_layout``."""
    import torch
    if X.dtype not in (torch.float32, torch.float64):
        raise TypeError(f"{what} must be float32 or float64, not {X.dtype}")
    if X.device.index != obj._scalar("device"):
        raise ValueError(f"{what} is on {X.device}, the harmony object on cuda:{obj._scalar('device')}")
    X, ld = row_layout(X, X.shape[1])
    return X, ctypes.c_void_p(X.data_ptr()), DTYPE[str(X.dtype)[6:]], ld


def rows_on(obj, X, what):
    """A checked embedding -> (whether it came from the host, the tensor the library reads, its device_rows
    arguments).  Host rows are uploaded with ``to_device``."""
    host = not is_cuda_tensor(X)
    if host:
        X = to_device(obj, X)
    x, *args = device_rows(obj, X, what)
    return host, x, args


def device_of(obj):
    """The torch device of a harmony object."""
    import torch
    return torch.device("cuda", obj._scalar("device"))


def handle(device):
    """A harmony object on ``device`` (None: the current one) for a call that needs no setup."""
    from .harmony import harmony  # needs the CUDA extension; fails loudly when it is missing
    return harmony(device=device)


def call(obj, entry, *args):
    """The library function ``entry`` on ``obj``'s handle with ``args`` and the current torch stream of its device, on
    which the library orders the call; a status other than 0 raises with the library's message."""
    obj._check(getattr(obj._L, entry)(obj._h, *args, current_stream(device_of(obj))))


def codes_on(obj, codes):
    """Integer codes -> an int32 tensor on ``obj``'s device (a CUDA tensor must already be there)."""
    import torch
    device = device_of(obj)
    if not is_cuda_tensor(codes):
        codes = torch.as_tensor(np.ascontiguousarray(codes, dtype=np.int32)).to(device)
    if codes.device != device:
        raise ValueError(f"codes are on {codes.device}, the harmony object on {device}")
    return codes


def dense_on(obj, codes):
    """Optional codes (None stays None) -> a contiguous int32 tensor on ``obj``'s device."""
    return None if codes is None else codes_on(obj, codes).contiguous()


def ptr(t):
    """A tensor's device pointer, NULL for None."""
    return ctypes.c_void_p(None if t is None else t.data_ptr())


def download(host, *ts):
    """The outputs as the caller's inputs came: numpy arrays for a host caller, the tensors otherwise (None stays)."""
    return [t.cpu().numpy() if host and t is not None else t for t in ts]


def to_host(v):
    """A CUDA tensor -> its numpy copy; anything else -> a numpy array."""
    return v.cpu().numpy() if is_cuda_tensor(v) else np.asarray(v)


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


def factorise_for(column, X):
    """``factorise`` of a label column for the rows X: the codes go to a CUDA X's device."""
    return factorise(column, X.device if is_cuda_tensor(X) else None)


def code_sets(codes, n):
    """int32 codes [N] or [n_sets, N] of any values (numpy or a CUDA tensor) -> the same as [n_sets, N]."""
    if is_cuda_tensor(codes):
        import torch
        if codes.dtype != torch.int32:
            raise TypeError(f"CUDA codes must be int32, not {codes.dtype}")
    else:
        codes = np.asarray(codes)
        if codes.dtype.kind not in "iu":
            raise TypeError(f"codes must be integers, not {codes.dtype}")
        if codes.size and (codes.min() < -2 ** 31 or codes.max() >= 2 ** 31):
            raise ValueError("codes must fit int32")
    if codes.ndim == 1:
        codes = codes[None]
    if codes.ndim != 2 or codes.shape[0] < 1 or codes.shape[1] != n:
        raise ValueError(f"codes must be [{n}] or [n_sets, {n}] with n_sets >= 1, not {tuple(codes.shape)}")
    return codes


def dense_codes(codes, n, what):
    """Codes 0..2^31 - 2 [N] (numpy or an int32 CUDA tensor) -> the same, and their count (largest + 1)."""
    if is_cuda_tensor(codes):
        import torch
        if codes.dtype != torch.int32:
            raise TypeError(f"CUDA {what} must be int32, not {codes.dtype}")
        if codes.ndim != 1 or codes.shape[0] != n:
            raise ValueError(f"{what} must be [{n}], not {tuple(codes.shape)}")
        return codes, int(codes.max()) + 1 if n else 0
    codes = np.asarray(codes)
    if codes.dtype.kind not in "iu":
        raise TypeError(f"{what} must be integers, not {codes.dtype}")
    if codes.ndim != 1 or codes.shape[0] != n:
        raise ValueError(f"{what} must be [{n}], not {codes.shape}")
    if codes.size and (codes.min() < 0 or codes.max() >= 2 ** 31 - 1):
        raise ValueError(f"{what} must be codes in 0..2^31 - 2")
    return codes, int(codes.max()) + 1 if n else 0


def missing(a):
    """Whether a host label array holds a missing value (NaN, None, pandas' NA / NaT)."""
    if a.dtype.kind == "f":
        return bool(np.isnan(a).any())
    if a.dtype.kind == "O":
        return any(v is None or (isinstance(v, float) and v != v) or type(v).__name__ in ("NAType", "NaTType") for v in a)
    return False


def _column(v):
    return v if is_cuda_tensor(v) else np.asarray(v)


def as_columns(meta_data, n_hint):
    """meta_data -> dict name -> 1-D array (CUDA tensors stay where they are).  Accepts a dict, a pandas DataFrame
    or one vector (R/ui.R:157-165: a bare vector becomes data.frame(batch_variable = ...))."""
    if hasattr(meta_data, "columns") and hasattr(meta_data, "__getitem__") and not isinstance(meta_data, dict):
        return {str(c): np.asarray(meta_data[c]) for c in meta_data.columns}, None
    if isinstance(meta_data, dict):
        return {str(k): _column(v) for k, v in meta_data.items()}, None
    v = _column(meta_data)
    if v.ndim == 1 and len(v) in n_hint:
        return {"batch_variable": v}, "batch_variable"
    raise ValueError("meta_data must be either a data.frame or a vector with batch values for each cell")


def label_device(cols, vars_use, data_mat, on_device):
    """The device of the used label columns that are CUDA tensors (None: all are host arrays).  They must be integer
    or bool tensors on data_mat's device."""
    device = None
    for v in vars_use:
        col = cols[v]
        if not is_cuda_tensor(col):
            continue
        import torch
        if col.dtype not in (torch.bool, torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64):
            raise TypeError(f"labels {v!r} on the GPU must be an integer or bool tensor, not {col.dtype}")
        if not on_device:
            raise ValueError(f"labels {v!r} are a CUDA tensor but data_mat is not: device labels go with a device "
                             f"embedding")
        if col.device != data_mat.device:
            raise ValueError(f"labels {v!r} are on {col.device}, data_mat on {data_mat.device}")
        if col.ndim != 1:
            raise ValueError(f"labels {v!r} must be a vector")
        device = col.device
    return device


def label_vector(v, n, what):
    """One label per row of an n-row embedding, none missing -> a numpy array, or the CUDA tensor as it is."""
    v = _column(v)
    if v.ndim != 1 or len(v) != n:
        raise ValueError(f"{what} must hold one label per row of X ({n})")
    if not is_cuda_tensor(v) and missing(v):
        raise ValueError(f"{what} holds missing labels")
    return v


def label_columns(meta_data, names, X):
    """The label columns ``names`` of ``meta_data`` (a DataFrame or a dict of columns) for the rows of the checked
    embedding ``X`` -> their arrays; a CUDA column must be an integer tensor on a CUDA ``X``'s device."""
    if not isinstance(meta_data, dict) and not hasattr(meta_data, "columns"):
        raise ValueError("meta_data must be a DataFrame or a dict of columns")
    cols, _ = as_columns(meta_data, ())
    for v in names:
        if v not in cols:
            raise ValueError(f"meta_data has no column {v!r}")
        label_vector(cols[v], X.shape[0], f"column {v!r}")
    label_device(cols, names, X, is_cuda_tensor(X))
    return [cols[v] for v in names]
