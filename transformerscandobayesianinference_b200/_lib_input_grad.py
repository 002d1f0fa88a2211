"""ctypes binding of the input-gradient entry points of libpfn_b200.so (include/pfn_b200_input_grad.h).

That header extends the C ABI of include/pfn_b200.h without changing it, and this module extends `_lib` the same way: it
restates the header's descriptor and five prototypes, gives them to the handle `_lib.load()` returns on first use, and
launches through `_lib._call` (so the launches count in `_lib.launch_count()`) behind `_lib._guarded`.
tests/test_input_grad_cabi_host.py holds the struct and prototypes against the header and each wrapper's calls against a
recorded log.
"""
import ctypes
from ctypes import POINTER

from . import _lib as L
from ._lib_ragged import _check_n_keys

c_int, c_void_p = ctypes.c_int, ctypes.c_void_p


class AttnCtxGradDesc(ctypes.Structure):
    _fields_ = [
        ("c", L.AttnCtxDesc),
        ("n_keys", c_void_p),
        ("lse", c_void_p),
        ("dout", c_void_p), ("ld_dout", c_int),
        ("dqkv", c_void_p), ("ld_dqkv", c_int),
        ("delta", c_void_p),
    ]


_P = c_void_p
# argument types of every entry point of include/pfn_b200_input_grad.h, in header order; each returns an int status
_PROTOTYPES = {
    "pfn_attention_ctx_grad_fwd_simt": [POINTER(AttnCtxGradDesc), c_void_p],
    "pfn_attention_ctx_grad_fwd_tc": [POINTER(AttnCtxGradDesc), c_void_p],
    "pfn_attention_ctx_bwd_simt": [POINTER(AttnCtxGradDesc), c_void_p],
    "pfn_attention_ctx_bwd_tc": [POINTER(AttnCtxGradDesc), c_void_p],
    "pfn_embed_input_bwd": [_P, c_int, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P, c_void_p],
}
EXPORTED_SYMBOLS = tuple(_PROTOTYPES)


def declare(lib):
    """Check that the ctypes handle `lib` exports every input-gradient entry point and give each its prototype; returns
    `lib`."""
    for name, argtypes in _PROTOTYPES.items():
        if not hasattr(lib, name):
            raise RuntimeError(f"libpfn_b200.so does not export {name}")
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = c_int
    return lib


_declared = []      # the handles declare() has been applied to


def _call(name, *args, launches=1):
    lib = L.load()
    if not any(h is lib for h in _declared):
        _declared.append(declare(lib))
    L._call(name, *args, launches=launches)


def _ctx_desc(qkv, kv, out, lse, m, n, B, H, dh, n_keys, who):
    if qkv.dtype != out.dtype or (n > 0 and kv.dtype != qkv.dtype):
        raise TypeError(f"{who}: qkv, kv and out must share one dtype")
    if n_keys is not None:
        _check_n_keys(n_keys, B, who)
    d = AttnCtxGradDesc()
    d.c = L.attention_ctx_desc(qkv, kv, out, m, n, B, H, dh)
    d.n_keys = None if n_keys is None else n_keys.data_ptr()
    d.lse = lse.data_ptr()
    return d


def attention_ctx_grad_fwd(qkv, kv, out, lse, m, n, B, H, dh, n_keys=None, use_tc=None):
    """_lib.attention_ctx_fwd (or, with n_keys, _lib_ragged.attention_ctx_ragged_fwd) that also writes lse [B*H, m] fp32
    for attention_ctx_bwd; out is the same bit for bit.  kv unused when n == 0."""
    _attention_ctx_grad_fwd(qkv, kv if n > 0 else None, out, lse, m, n, B, H, dh, n_keys, use_tc)


@L._guarded
def _attention_ctx_grad_fwd(qkv, kv, out, lse, m, n, B, H, dh, n_keys, use_tc):
    d = _ctx_desc(qkv, kv, out, lse, m, n, B, H, dh, n_keys, "attention_ctx_grad_fwd")
    if use_tc is None:
        use_tc = L.tc_attention_ok(qkv, dh)
    _call("pfn_attention_ctx_grad_fwd_tc" if use_tc else "pfn_attention_ctx_grad_fwd_simt", ctypes.byref(d))


def attention_ctx_bwd(qkv, kv, out, lse, dout, dqkv, delta, m, n, B, H, dh, n_keys=None, use_tc=None):
    """The backward of attention_ctx_grad_fwd: dqkv [m*B, 3*H*dh] written completely (dQ, and dK / dV of each row's own
    key); the cached kv is a constant and gets no gradient.  delta: [B*H, m] fp32 scratch."""
    _attention_ctx_bwd(qkv, kv if n > 0 else None, out, lse, dout, dqkv, delta, m, n, B, H, dh, n_keys, use_tc)


@L._guarded
def _attention_ctx_bwd(qkv, kv, out, lse, dout, dqkv, delta, m, n, B, H, dh, n_keys, use_tc):
    d = _ctx_desc(qkv, kv, out, lse, m, n, B, H, dh, n_keys, "attention_ctx_bwd")
    if dout.dtype != qkv.dtype or dqkv.dtype != qkv.dtype:
        raise TypeError("attention_ctx_bwd: dout and dqkv must have the dtype of qkv")
    d.dout, d.ld_dout = dout.data_ptr(), dout.stride(0)
    d.dqkv, d.ld_dqkv = dqkv.data_ptr(), dqkv.stride(0)
    d.delta = delta.data_ptr()
    if use_tc is None:
        use_tc = L.tc_attention_ok(qkv, dh)
    # the tensor-core backward runs the delta pass and the dQ kernel; the fp32-FMA one forms delta inside its dQ kernel
    _call("pfn_attention_ctx_bwd_tc" if use_tc else "pfn_attention_ctx_bwd_simt", ctypes.byref(d),
          launches=2 if use_tc else 1)


@L._guarded
def embed_input_bwd(dout, Wx, wy, dx, dy, T, B, F, E, sep, n_keys=None):
    """dx [T*B, F] = dout Wx and dy [T*B] = dout . wy on the rows t < sep (t < n_keys[b] of dataset b when n_keys is
    given), 0 elsewhere; both fp32, overwritten.  F <= 64."""
    if n_keys is not None:
        _check_n_keys(n_keys, B, "embed_input_bwd")
    _call("pfn_embed_input_bwd", L.ptr(dout), L.dtype_code(dout), L.ptr(Wx), L.ptr(wy), L.ptr(dx), L.ptr(dy), T, B, F, E,
          sep, L.ptr(n_keys))
