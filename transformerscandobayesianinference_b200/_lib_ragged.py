"""ctypes binding of the ragged-dataset attention entry points of libpfn_b200.so (include/pfn_b200_ragged.h).

That header extends the C ABI of include/pfn_b200.h without changing it, and this module extends `_lib` the same way: it
restates the header's two descriptors and four prototypes, gives them to the handle `_lib.load()` returns on first use,
and launches through `_lib._call` (so the launches count in `_lib.launch_count()`) behind `_lib._guarded`.
tests/test_ragged_cabi_host.py holds the structs and prototypes against the header and each wrapper's calls against a
recorded log.
"""
import ctypes
from ctypes import POINTER

import torch

from . import _lib as L

c_int, c_float, c_void_p = ctypes.c_int, ctypes.c_float, ctypes.c_void_p


class AttnRaggedDesc(ctypes.Structure):
    _fields_ = [
        ("T", c_int), ("B", c_int), ("H", c_int), ("dh", c_int),
        ("dtype", c_int), ("scale", c_float),
        ("qkv", c_void_p), ("ld_qkv", c_int),
        ("out", c_void_p), ("ld_out", c_int),
        ("n_keys", c_void_p),
    ]


class AttnCtxRaggedDesc(ctypes.Structure):
    _fields_ = [
        ("m", c_int), ("n", c_int), ("B", c_int), ("H", c_int), ("dh", c_int),
        ("dtype", c_int), ("scale", c_float),
        ("qkv", c_void_p), ("ld_qkv", c_int),
        ("kv", c_void_p), ("ld_kv", c_int),
        ("out", c_void_p), ("ld_out", c_int),
        ("n_keys", c_void_p),
    ]


# argument types of every entry point of include/pfn_b200_ragged.h, in header order; each returns an int status
_PROTOTYPES = {
    "pfn_attention_ragged_fwd_simt": [POINTER(AttnRaggedDesc), c_void_p],
    "pfn_attention_ragged_fwd_tc": [POINTER(AttnRaggedDesc), c_void_p],
    "pfn_attention_ctx_ragged_fwd_simt": [POINTER(AttnCtxRaggedDesc), c_void_p],
    "pfn_attention_ctx_ragged_fwd_tc": [POINTER(AttnCtxRaggedDesc), c_void_p],
}
EXPORTED_SYMBOLS = tuple(_PROTOTYPES)


def declare(lib):
    """Check that the ctypes handle `lib` exports every ragged entry point and give each its prototype; returns `lib`."""
    for name, argtypes in _PROTOTYPES.items():
        if not hasattr(lib, name):
            raise RuntimeError(f"libpfn_b200.so does not export {name}")
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = c_int
    return lib


_declared = []      # the handles declare() has been applied to


def _call(name, desc):
    lib = L.load()
    if not any(h is lib for h in _declared):
        _declared.append(declare(lib))
    L._call(name, ctypes.byref(desc))


def _check_n_keys(n_keys, B, who):
    """n_keys: the int32 [B] device tensor of per-dataset key counts."""
    if n_keys.dtype != torch.int32 or n_keys.shape != (B,) or not n_keys.is_contiguous():
        raise TypeError(f"{who}: n_keys must be a contiguous int32 tensor of shape ({B},), got {n_keys.dtype} "
                        f"{tuple(n_keys.shape)}")


@L._guarded
def attention_ragged_fwd(qkv, out, T, B, H, dh, n_keys, use_tc=None):
    """out [T*B, H*dh] <- the masked attention of packed qkv [T*B, 3*H*dh] where dataset b's keys are its rows
    [0, n_keys[b]) and rows t >= n_keys[b] also attend to themselves (no lse).  n_keys: int32 [B] on the device."""
    _check_n_keys(n_keys, B, "attention_ragged_fwd")
    d = AttnRaggedDesc()
    d.T, d.B, d.H, d.dh = T, B, H, dh
    d.dtype = L.dtype_code(qkv)
    d.scale = 1.0 / (dh ** 0.5)
    d.qkv, d.ld_qkv = qkv.data_ptr(), qkv.stride(0)
    d.out, d.ld_out = out.data_ptr(), out.stride(0)
    d.n_keys = n_keys.data_ptr()
    if use_tc is None:
        use_tc = L.tc_attention_ok(qkv, dh)
    _call("pfn_attention_ragged_fwd_tc" if use_tc else "pfn_attention_ragged_fwd_simt", d)


def attention_ctx_ragged_fwd(qkv, kv, out, m, n, B, H, dh, n_keys, use_tc=None):
    """_lib.attention_ctx_fwd where the query rows of dataset b attend to its first n_keys[b] cached rows only (and to
    themselves); n_keys: int32 [B] on the device, kv unused when n == 0."""
    _attention_ctx_ragged_fwd(qkv, kv if n > 0 else None, out, m, n, B, H, dh, n_keys, use_tc)   # an unread kv is not checked


@L._guarded
def _attention_ctx_ragged_fwd(qkv, kv, out, m, n, B, H, dh, n_keys, use_tc):
    if qkv.dtype != out.dtype or (n > 0 and kv.dtype != qkv.dtype):
        raise TypeError("attention_ctx_ragged_fwd: qkv, kv and out must share one dtype")
    _check_n_keys(n_keys, B, "attention_ctx_ragged_fwd")
    d = AttnCtxRaggedDesc()
    d.m, d.n, d.B, d.H, d.dh = m, n, B, H, dh
    d.dtype = L.dtype_code(qkv)
    d.scale = 1.0 / (dh ** 0.5)
    d.qkv, d.ld_qkv = qkv.data_ptr(), qkv.stride(0)
    d.kv, d.ld_kv = (kv.data_ptr(), kv.stride(0)) if n > 0 else (None, 0)
    d.out, d.ld_out = out.data_ptr(), out.stride(0)
    d.n_keys = n_keys.data_ptr()
    if use_tc is None:
        use_tc = L.tc_attention_ok(qkv, dh)
    _call("pfn_attention_ctx_ragged_fwd_tc" if use_tc else "pfn_attention_ctx_ragged_fwd_simt", d)
