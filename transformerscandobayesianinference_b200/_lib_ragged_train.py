"""ctypes binding of the ragged-dataset training entry points of libpfn_b200.so (include/pfn_b200_ragged_train.h).

That header extends the C ABI of include/pfn_b200.h without changing it, and this module extends `_lib` the same way:
it restates the header's descriptor and six prototypes, gives them to the handle `_lib.load()` returns on first use, and
launches through `_lib._call` (so the launches count in `_lib.launch_count()`) behind `_lib._guarded`.
tests/test_ragged_train_cabi_host.py holds the struct and prototypes against the header and each wrapper's calls against
a recorded log.
"""
import ctypes
from ctypes import POINTER

from . import _lib as L
from ._lib_ragged import _check_n_keys

c_int, c_void_p = ctypes.c_int, ctypes.c_void_p


class AttnRaggedTrainDesc(ctypes.Structure):
    _fields_ = [
        ("a", L.AttnDesc),
        ("n_keys", c_void_p),
    ]


_P = c_void_p
# argument types of every entry point of include/pfn_b200_ragged_train.h, in header order; each returns an int status
_PROTOTYPES = {
    "pfn_attention_ragged_train_fwd_simt": [POINTER(AttnRaggedTrainDesc), c_void_p],
    "pfn_attention_ragged_train_fwd_tc": [POINTER(AttnRaggedTrainDesc), c_void_p],
    "pfn_attention_ragged_train_bwd_simt": [POINTER(AttnRaggedTrainDesc), c_void_p],
    "pfn_attention_ragged_train_bwd_tc": [POINTER(AttnRaggedTrainDesc), c_void_p],
    "pfn_embed_ragged_fwd": [_P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P, c_void_p],
    "pfn_embed_ragged_bwd": [_P, c_int, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, _P, c_void_p],
}
EXPORTED_SYMBOLS = tuple(_PROTOTYPES)


def declare(lib):
    """Check that the ctypes handle `lib` exports every ragged training entry point and give each its prototype;
    returns `lib`."""
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


def _desc(a, n_keys, B, who):
    _check_n_keys(n_keys, B, who)
    d = AttnRaggedTrainDesc()
    d.a = a
    d.n_keys = n_keys.data_ptr()
    return d


@L._guarded
def attention_ragged_train_fwd(qkv, out, lse, T, B, H, dh, sep_max, n_keys, use_tc=None, drop=None):
    """_lib.attention_fwd where dataset b has the separator n_keys[b] (int32 [B] on the device, each in [0, sep_max]):
    its row i attends to rows [0, n_keys[b]) and, when i >= n_keys[b], to itself.  Writes out and lse."""
    d = _desc(L.attention_desc(qkv, out, lse, T, B, H, dh, sep_max, drop=drop), n_keys, B, "attention_ragged_train_fwd")
    if use_tc is None:
        use_tc = L.tc_attention_ok(qkv, dh)
    _call("pfn_attention_ragged_train_fwd_tc" if use_tc else "pfn_attention_ragged_train_fwd_simt", ctypes.byref(d))


@L._guarded
def attention_ragged_train_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, dh, sep_max, n_keys, use_tc=None, drop=None,
                               dq_colsum=None, delta_token_major=False):
    """_lib.attention_bwd of attention_ragged_train_fwd: dqkv [T*B, 3*H*dh] written completely."""
    d = _desc(L.attention_desc(qkv, out, lse, T, B, H, dh, sep_max, dout, dqkv, delta, drop=drop), n_keys, B,
              "attention_ragged_train_bwd")
    if use_tc is None:
        use_tc = L.tc_attention_ok(qkv, dh)
    if dq_colsum is not None:
        assert use_tc, "dq_colsum is produced by the tensor-core backward only"
        d.a.dq_colsum = dq_colsum.data_ptr()
    if delta_token_major:
        assert use_tc, "a precomputed token-major delta is consumed by the tensor-core backward only"
        d.a.delta_token_major = 1
    _call("pfn_attention_ragged_train_bwd_tc" if use_tc else "pfn_attention_ragged_train_bwd_simt", ctypes.byref(d),
          launches=2)


@L._guarded
def embed_ragged_fwd(x, y, Wx, bx, wy, by, out, T, B, F, E, n_keys):
    """_lib.embed_fwd with the y embedding on the rows t < n_keys[b] of dataset b."""
    _check_n_keys(n_keys, B, "embed_ragged_fwd")
    _call("pfn_embed_ragged_fwd", L.ptr(x), L.ptr(y), L.ptr(Wx), L.ptr(bx), L.ptr(wy), L.ptr(by), L.ptr(out),
          L.dtype_code(out), T, B, F, E, L.ptr(n_keys))


@L._guarded
def embed_ragged_bwd(dout, x, y, dWx, dbx, dwy, dby, T, B, F, E, n_keys):
    """_lib.embed_bwd with dwy, dby summed over the rows t < n_keys[b] of dataset b."""
    _check_n_keys(n_keys, B, "embed_ragged_bwd")
    _call("pfn_embed_ragged_bwd", L.ptr(dout), L.dtype_code(dout), L.ptr(x), L.ptr(y), L.ptr(dWx), L.ptr(dbx),
          L.ptr(dwy), L.ptr(dby), T, B, F, E, L.ptr(n_keys), launches=(F + 7) // 8)
