"""ctypes binding of libpfn_b200.so (the C ABI declared in include/pfn_b200.h).

There is deliberately no fallback: if the shared object is missing or a call fails, a RuntimeError with the
library's own message is raised.  Tensors are passed as raw device pointers on torch's current CUDA stream.

The header is restated here once: one ctypes Structure per descriptor, the mirrored enum constants, and one
`_PROTOTYPES` line per entry point.  tests/test_cabi.py holds all three against the header.

Each launching entry point has one thin wrapper below.  `@_guarded` rejects a tensor argument that is not on the call's
one CUDA device before anything else happens and makes that device current; the wrapper body turns its arguments into
the C arguments (`ptr`, `dtype_code`, `_set_ptrs` for descriptor pointer fields, `_u32` for seeds) and launches through
`_call`, which counts the launches, passes torch's current stream and raises on a failed call.
tests/test_lib_calls_host.py holds every wrapper's calls against a recorded log.
"""
import ctypes
import functools
import os
from ctypes import POINTER

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# PFN_B200_LIB points at another build of the same library (A/B measurements of kernel variants); default: the in-tree build
LIB_PATH = os.environ.get("PFN_B200_LIB") or os.path.join(_HERE, "libpfn_b200.so")

F32, BF16 = 0, 1
EPI_NONE, EPI_GELU, EPI_GELU_BWD, EPI_ROWDOT, EPI_MUL = 0, 1, 2, 3, 4
KERNEL_RBF, KERNEL_MATERN12, KERNEL_MATERN32, KERNEL_MATERN52 = 0, 1, 2, 3

c_int, c_uint32, c_float, c_double, c_void_p = ctypes.c_int, ctypes.c_uint32, ctypes.c_float, ctypes.c_double, ctypes.c_void_p


class GemmDesc(ctypes.Structure):
    _fields_ = [
        ("M", c_int), ("N", c_int), ("K", c_int),
        ("A", c_void_p), ("lda", c_int), ("a_mn_major", c_int),
        ("B", c_void_p), ("ldb", c_int), ("b_mn_major", c_int),
        ("C", c_void_p), ("ldc", c_int), ("c_dtype", c_int),
        ("bias", c_void_p),
        ("aux", c_void_p), ("ld_aux", c_int),
        ("C2", c_void_p), ("ldc2", c_int),
        ("epilogue", c_int), ("accumulate", c_int), ("k_splits", c_int), ("ab_dtype", c_int),
        ("rowdot_out", c_void_p), ("rowdot_width", c_int), ("c2_gelu_grad", c_int),
    ]


class StrokeDesc(ctypes.Structure):
    _fields_ = [(n, c_int) for n in ("S", "C", "strokes_min", "strokes_max", "len_min", "len_max", "start_min", "start_max",
                                     "width_min", "width_max", "offset_min", "offset_max", "jitter_min", "jitter_max",
                                     "max_iters")]


STROKE_MAX_STROKES, STROKE_MAX_SIDE = 16, 112


class OmniglotDesc(ctypes.Structure):
    _fields_ = [(n, c_int) for n in ("S", "n_classes", "B", "n_way", "k_shot", "T", "jonas", "train", "translate", "pool_lo",
                                     "pool_n", "n_alpha", "alpha_min")]


OMNIGLOT_IMAGES, OMNIGLOT_MAX_WAY, OMNIGLOT_MAX_SIDE = 20, 64, 105


class AdamTensor(ctypes.Structure):
    _fields_ = [("p", c_void_p), ("g", c_void_p), ("m", c_void_p), ("v", c_void_p), ("p_bf16", c_void_p),
                ("n", ctypes.c_longlong)]


class GpFitDesc(ctypes.Structure):
    _fields_ = [
        ("B", c_int), ("T", c_int), ("F", c_int),
        ("x", c_void_p), ("y", c_void_p),
        ("n_ts", c_int), ("ts", POINTER(c_int)),
        ("kernel_type", c_int),
        ("ls_conc", c_double), ("ls_rate", c_double), ("os_conc", c_double), ("os_rate", c_double),
        ("noise_conc", c_double), ("noise_rate", c_double),
        ("noise_lb", c_double),
        ("theta0", c_void_p), ("noise_init", c_double),
        ("max_iter", c_int), ("max_eval", c_int),
        ("ftol", c_double), ("gtol", c_double),
        ("theta", c_void_p), ("f", c_void_p), ("grad", c_void_p), ("mean", c_void_p), ("var", c_void_p),
        ("iters", c_void_p), ("nevals", c_void_p), ("status", c_void_p),
    ]


GP_FIT_MAX_T, GP_FIT_MAX_F = 128, 32
GP_FIT_CONVERGED, GP_FIT_MAX_ITER, GP_FIT_LINE_SEARCH, GP_FIT_NOT_PD = 0, 1, 2, 3


class GpMcmcDesc(ctypes.Structure):
    _fields_ = [
        ("B", c_int), ("T", c_int), ("F", c_int),
        ("x", c_void_p), ("y", c_void_p),
        ("n_ts", c_int), ("ts", POINTER(c_int)),
        ("kernel_type", c_int),
        ("ls_conc", c_double), ("ls_rate", c_double), ("os_conc", c_double), ("os_rate", c_double),
        ("noise_conc", c_double), ("noise_rate", c_double),
        ("num_samples", c_int), ("warmup_steps", c_int), ("max_tree_depth", c_int), ("n_pred", c_int),
        ("seed", c_uint32),
        ("init", c_void_p),
        ("samples", c_void_p), ("log_samples", c_void_p), ("mean", c_void_p), ("var", c_void_p), ("potential", c_void_p), ("grad", c_void_p),
        ("step_size", c_void_p), ("accept", c_void_p), ("diag", c_void_p), ("trace", c_void_p),
    ]


GP_MCMC_MAX_DEPTH = 10
GP_MCMC_DIAG_NAMES = ("leapfrog", "evals", "div_warmup", "div_sampling", "max_depth_hits", "not_pd")   # diag columns


class BnnMcmcDesc(ctypes.Structure):
    _fields_ = [
        ("N", c_int), ("n", c_int), ("n_test", c_int), ("F", c_int), ("E", c_int),
        ("x_train", c_void_p), ("y_train", c_void_p), ("x_test", c_void_p),
        ("num_samples", c_int), ("warmup_steps", c_int), ("max_tree_depth", c_int),
        ("seed", c_uint32),
        ("init", c_void_p),
        ("samples", c_void_p), ("probs", c_void_p), ("obs", c_void_p), ("potential", c_void_p), ("grad", c_void_p),
        ("step_size", c_void_p), ("accept", c_void_p), ("diag", c_void_p), ("trace", c_void_p), ("workspace", c_void_p),
    ]


BNN_MAX_D, BNN_MAX_N = 1024, 1024


class KnnCvDesc(ctypes.Structure):
    _fields_ = [
        ("S", c_int), ("n", c_int), ("m", c_int), ("F", c_int),
        ("x", c_void_p), ("y", c_void_p),
        ("proba", c_void_p), ("k_best", c_void_p), ("cv_mean", c_void_p), ("status", c_void_p),
    ]


KNN_MAX_N, KNN_MAX_F, KNN_MAX_K = 1024, 1024, 5
KNN_OK, KNN_BAD_LABEL, KNN_FEW_MEMBERS, KNN_ONE_CLASS = 0, 1, 2, 3


class AttnDesc(ctypes.Structure):
    _fields_ = [
        ("T", c_int), ("B", c_int), ("H", c_int), ("dh", c_int), ("sep", c_int),
        ("dtype", c_int), ("scale", c_float),
        ("qkv", c_void_p), ("ld_qkv", c_int),
        ("out", c_void_p), ("ld_out", c_int),
        ("lse", c_void_p),
        ("dout", c_void_p), ("ld_dout", c_int),
        ("dqkv", c_void_p), ("ld_dqkv", c_int),
        ("delta", c_void_p), ("batch_major", c_int),
        ("drop_seed", c_uint32), ("drop_thr", c_int),
        ("dq_colsum", c_void_p), ("delta_token_major", c_int),
    ]


class AttnCtxDesc(ctypes.Structure):
    _fields_ = [
        ("m", c_int), ("n", c_int), ("B", c_int), ("H", c_int), ("dh", c_int),
        ("dtype", c_int), ("scale", c_float),
        ("qkv", c_void_p), ("ld_qkv", c_int),
        ("kv", c_void_p), ("ld_kv", c_int),
        ("out", c_void_p), ("ld_out", c_int),
    ]


class ConvDesc(ctypes.Structure):
    _fields_ = [
        ("N", c_int), ("S", c_int), ("C_in", c_int), ("dtype", c_int),
        ("x", c_void_p), ("w", c_void_p), ("bias", c_void_p), ("g", c_void_p), ("y", c_void_p),
        ("dw", c_void_p), ("db", c_void_p), ("workspace", c_void_p),
    ]


CONV_MAX_SIDE, CONV_CH = 112, 64


class RidgePrefixDesc(ctypes.Structure):
    _fields_ = [
        ("B", c_int), ("T", c_int), ("F", c_int),
        ("alpha", c_double),
        ("x", c_void_p), ("y", c_void_p), ("target", c_void_p),
        ("pred", c_void_p), ("sq_err", c_void_p),
    ]


RIDGE_MAX_F = 64


class ExactGpDesc(ctypes.Structure):
    _fields_ = [
        ("B", c_int), ("T", c_int), ("F", c_int),
        ("mode", c_int),
        ("length_scale", c_double), ("alpha", c_double),
        ("x", c_void_p), ("y", c_void_p), ("z", c_void_p),
        ("mean", c_void_p), ("var", c_void_p), ("status", c_void_p),
        ("sample", c_void_p), ("rank", c_void_p), ("factor", c_void_p), ("perm", c_void_p),
    ]


EXACT_GP_EVALUATE, EXACT_GP_SAMPLE = 0, 1
HEAD_TEMPS = 10        # temperature logits of decoders.ScaledDecoder


P, I, F, U = c_void_p, c_int, c_float, c_uint32

# argument types of every entry point, in header order, one per C parameter (pointers to descriptors as POINTER(...), every
# other pointer, the stream included, as P).  Each returns an int status, except pfn_last_error (a string).
_PROTOTYPES = {
    "pfn_last_error": [],
    "pfn_version": [],
    "pfn_num_sms": [],
    "pfn_gemm_bf16_tc": [POINTER(GemmDesc), P],
    "pfn_gemm_simt": [POINTER(GemmDesc), P],
    "pfn_attention_fwd_simt": [POINTER(AttnDesc), P],
    "pfn_attention_bwd_simt": [POINTER(AttnDesc), P],
    "pfn_attention_fwd_tc": [POINTER(AttnDesc), P],
    "pfn_attention_bwd_tc": [POINTER(AttnDesc), P],
    "pfn_attention_ctx_fwd_simt": [POINTER(AttnCtxDesc), P],
    "pfn_attention_ctx_fwd_tc": [POINTER(AttnCtxDesc), P],
    "pfn_embed_fwd": [P, P, P, P, P, P, P, I, I, I, I, I, I, P],
    "pfn_embed_bwd": [P, I, P, P, P, P, P, P, I, I, I, I, I, P],
    "pfn_layernorm_fwd": [P, I, P, P, P, I, P, P, I, I, F, I, P],
    "pfn_layernorm_bwd": [P, I, P, I, P, P, P, P, I, P, P, P, I, I, I, P],
    "pfn_dropout": [P, I, P, I, P, I, I, I, I, U, I, P],
    "pfn_dropout_keep_mask": [P, I, I, U, I, P],
    "pfn_adam_chunk_elems": [],
    "pfn_adam_step": [P, P, I, I, F, F, F, F, F, F, I, P, P],
    "pfn_colsum": [P, I, I, P, I, I, P],
    "pfn_bar_nll_fwd": [P, I, I, P, P, I, I, P, P, P, P, I, P],
    "pfn_bar_nll_bwd": [P, I, I, P, P, P, P, I, I, I, I, I, P],
    "pfn_bar_bucket_idx": [P, P, I, P, I, P],
    "pfn_gp_sample": [P, P, P, P, P, F, I, P, P, P, I, I, I, P],
    "pfn_gp_fit": [POINTER(GpFitDesc), P],
    "pfn_gp_mcmc": [POINTER(GpMcmcDesc), P],
    "pfn_stroke_geometry": [POINTER(StrokeDesc), U, I, P, P, P, P],
    "pfn_stroke_render": [POINTER(StrokeDesc), U, P, P, P, P, I, I, I, P],
    "pfn_stroke_raster": [P, P, P, P, P, P, I, I, I, P],
    "pfn_omniglot_episodes": [POINTER(OmniglotDesc), U, P, P, P, P, P, P],
    "pfn_bnn_prior": [U, I, I, I, I, I, P, P, P, P, P, P],
    "pfn_bnn_mcmc_workspace": [POINTER(BnnMcmcDesc)],
    "pfn_bnn_mcmc": [POINTER(BnnMcmcDesc), P],
    "pfn_knn_cv": [POINTER(KnnCvDesc), P],
    "pfn_conv_fwd": [POINTER(ConvDesc), P],
    "pfn_conv_dgrad": [POINTER(ConvDesc), P],
    "pfn_conv_wgrad_workspace": [POINTER(ConvDesc)],
    "pfn_conv_wgrad": [POINTER(ConvDesc), P],
    "pfn_conv_mean_fwd": [P, I, I, I, P, P],
    "pfn_conv_mean_bwd": [P, P, I, I, I, P, P],
    "pfn_ridge_prefix": [POINTER(RidgePrefixDesc), P],
    "pfn_exact_gp": [POINTER(ExactGpDesc), P],
    "pfn_scaled_head_fwd": [P, I, I, P, I, P, I, P],
    "pfn_scaled_head_bwd": [P, I, P, I, P, I, P, I, I, I, I, P],
    "pfn_fixed_scaled_head_fwd": [P, I, I, P, I, P, I, P, I, P],
    "pfn_fixed_scaled_head_bwd": [P, I, P, I, P, I, P, I, I, I, P, P, I, I, P],
}
EXPORTED_SYMBOLS = tuple(_PROTOTYPES)

_lib = None
_launches = 0          # kernel launches issued through this binding (bench.py reports it as gpu_launches)
PROFILE_GEMM = None    # when a list: (flops, start_event, end_event, algorithmic operand+result bytes) is appended for every wgmma GEMM launch


_NUM_SMS = {}


def num_sms(device=None):
    """SM count of `device` (default: the current device) as the library sees it (grid sizing of the persistent kernels)."""
    idx = torch.cuda.current_device() if device is None else torch.device(device).index
    if idx not in _NUM_SMS:
        with torch.cuda.device(idx):
            _NUM_SMS[idx] = int(load().pfn_num_sms())
    return _NUM_SMS[idx]


def reset_launch_count():
    global _launches
    _launches = 0


def launch_count():
    return _launches


def declare(lib):
    """Check that the ctypes handle `lib` exports every entry point and give each its prototype; returns `lib`."""
    for name, argtypes in _PROTOTYPES.items():
        if not hasattr(lib, name):
            raise RuntimeError(f"libpfn_b200.so does not export {name}")
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = ctypes.c_char_p if name == "pfn_last_error" else c_int
    return lib


def load():
    """Load (once) and return the ctypes handle.  Raises if the library has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU / PyTorch fallback for the PFN hot path)")
        _lib = declare(ctypes.CDLL(LIB_PATH))
    return _lib


def check(rc, what):
    if rc != 0:
        msg = load().pfn_last_error()
        raise RuntimeError(f"{what} failed (rc={rc}): {msg.decode() if msg else 'no message'}")


def stream_ptr(device=None):
    """torch's current stream ON `device` (not on whatever device happens to be current)."""
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)


class on_device:
    """Make `device` the current CUDA device for the duration of a library call: the kernels launch on the current
    device, so a call whose tensors live elsewhere (train(gpu_device='cuda:1'), a rank's own GPU) must switch first."""
    __slots__ = ("idx", "prev")

    def __init__(self, device):
        self.idx = device.index if device.index is not None else torch.cuda.current_device()
        self.prev = None

    def __enter__(self):
        cur = torch.cuda.current_device()
        if cur != self.idx:
            self.prev = cur
            torch.cuda.set_device(self.idx)
        return self

    def __exit__(self, *exc):
        if self.prev is not None:
            torch.cuda.set_device(self.prev)
        return False


def dtype_code(t):
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.bfloat16:
        return BF16
    raise TypeError(f"unsupported dtype {t.dtype} (fp32 / bf16 only)")


def ptr(t):
    return None if t is None else c_void_p(t.data_ptr())


def require_cuda(*tensors):
    """All tensors must live on ONE CUDA device; returns that device."""
    dev = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError(
                "the PFN hot path runs on sm_90a CUDA kernels only; got a tensor on "
                f"{t.device}. Move the model and data to a CUDA device (no CPU fallback exists).")
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise RuntimeError(f"tensors of one kernel call live on different devices ({dev} and {t.device})")
    return dev


def cuda_device(device, what):
    """`device` with its index filled in; raises on a non-CUDA device.  `what` names the caller and its kernel."""
    dev = torch.device(device)
    if dev.type != 'cuda':
        raise RuntimeError(f"{what}; device {dev} is not a CUDA device (there is no CPU fallback)")
    return dev if dev.index is not None else torch.device('cuda', torch.cuda.current_device())


def compute_device(device, what):
    """Where a sampler runs: `device` when it is a CUDA device (index filled in), otherwise (a CPU device, or None) the
    current CUDA device, whose results the caller may copy to `device`.  Raises when there is no CUDA device."""
    if device is not None and torch.device(device).type == 'cuda':
        return cuda_device(device, what)
    if not torch.cuda.is_available():
        raise RuntimeError(f"{what}; no CUDA device is available (there is no CPU fallback)")
    return torch.device('cuda', torch.cuda.current_device())


def draw_seed(seed=None):
    """`seed`, or when None one draw of torch's CPU generator: reproducible under torch.manual_seed, no device sync.
    Seeds the counter-based random numbers of the samplers, the NUTS chains and dropout."""
    return int(torch.randint(0, 2 ** 31 - 1, (1,)).item()) if seed is None else int(seed)


_Tensor = torch.Tensor     # bound once: the guard below runs on every library call


def _guarded(fn):
    """Check that every tensor argument of the wrapped library call lives on one CUDA device (require_cuda), then run the
    call with that device current (so that `stream_ptr()`, `num_sms()` and the launch itself all refer to the device
    that owns the data).  The check comes first, so a rejected call neither reaches the library nor counts a launch.
    A keyword argument may also be a tuple holding a tensor (gemm's `rowdot`)."""
    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        tensors = [a for a in args if isinstance(a, _Tensor)]
        for v in kwargs.values():
            if isinstance(v, _Tensor):
                tensors.append(v)
            elif isinstance(v, tuple):
                tensors += [t for t in v if isinstance(t, _Tensor)]
        dev = require_cuda(*tensors)
        if dev is None:
            return fn(*args, **kwargs)
        with on_device(dev):
            return fn(*args, **kwargs)
    return wrapper


def _call(name, *args, launches=1):
    """Call entry point `name` with `args` and torch's current stream, adding the `launches` kernels it launches to
    launch_count(); raises the library's error when the call fails.  `name` is looked up on the handle at every call."""
    global _launches
    _launches += launches
    check(getattr(load(), name)(*(args + (stream_ptr(),))), name)     # one tuple: cheaper per call than f(*args, s)


def _workspace(name, desc):
    """The workspace size that query entry point `name` reports for `desc`; a negative size is the library's error."""
    n = int(getattr(load(), name)(ctypes.byref(desc)))
    if n < 0:
        check(1, name)
    return n


def _set_ptrs(d, **tensors):
    """Point each named field of the descriptor `d` at its tensor's data (None: NULL); returns `d`."""
    for name, t in tensors.items():
        setattr(d, name, None if t is None else t.data_ptr())
    return d


def _u32(seed):
    """`seed` as the library's uint32_t seeds take it: its low 32 bits (two's complement for a negative seed)."""
    return int(seed) & 0xFFFFFFFF


# ------------------------------------------------------------------------------------------------
# thin wrappers
# ------------------------------------------------------------------------------------------------
@_guarded
def gemm(A, B, C, *, a_mn_major=False, b_mn_major=False, bias=None, aux=None, C2=None, epilogue=EPI_NONE,
         accumulate=False, k_splits=1, M=None, N=None, K=None, use_tc=None, rowdot=None, c2_gelu_grad=False):
    """C[M,N] (+)= epi(A . B^T-ish + bias) (+ aux).  Operands are 2-D row-major tensors (stride(1) == 1)."""
    if M is None:
        M = A.shape[1] if a_mn_major else A.shape[0]
    if K is None:
        K = A.shape[0] if a_mn_major else A.shape[1]
    if N is None:
        N = B.shape[1] if b_mn_major else B.shape[0]
    d = GemmDesc()
    d.M, d.N, d.K = M, N, K
    d.A, d.lda, d.a_mn_major = A.data_ptr(), A.stride(0), int(a_mn_major)
    d.B, d.ldb, d.b_mn_major = B.data_ptr(), B.stride(0), int(b_mn_major)
    d.C, d.ldc, d.c_dtype = C.data_ptr(), C.stride(0), dtype_code(C)
    d.bias = bias.data_ptr() if bias is not None else None
    d.aux, d.ld_aux = (aux.data_ptr(), aux.stride(0)) if aux is not None else (None, 0)
    d.C2, d.ldc2 = (C2.data_ptr(), C2.stride(0)) if C2 is not None else (None, 0)
    d.epilogue, d.accumulate, d.k_splits = epilogue, int(accumulate), k_splits
    d.ab_dtype = dtype_code(A)
    d.c2_gelu_grad = int(bool(c2_gelu_grad))
    if rowdot is not None:       # (fp32 [M, N // width] zeroed tensor, width): EPI_ROWDOT target
        d.rowdot_out, d.rowdot_width = rowdot[0].data_ptr(), int(rowdot[1])
    if use_tc is None:
        use_tc = tc_gemm_ok(A, B, C, aux, C2)
    if not use_tc:
        _call("pfn_gemm_simt", ctypes.byref(d))
    elif PROFILE_GEMM is None:
        _call("pfn_gemm_bf16_tc", ctypes.byref(d))
    else:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _call("pfn_gemm_bf16_tc", ctypes.byref(d))
        e1.record()
        PROFILE_GEMM.append((2.0 * M * N * K, e0, e1, gemm_bytes(d)))


def gemm_bytes(d):
    """Algorithmic HBM bytes of the wgmma GEMM `d` (a GemmDesc): bf16 A and B read once, C (and C2) written once in C's
    dtype, bf16 aux read once."""
    esz = 4 if d.c_dtype == F32 else 2
    return 2.0 * (d.M * d.K + d.N * d.K) + esz * d.M * d.N * (2 if d.C2 else 1) + (2.0 * d.M * d.N if d.aux else 0.0)


def tc_gemm_ok(A, B, C, aux=None, C2=None):
    if A.dtype != torch.bfloat16 or B.dtype != torch.bfloat16:
        return False
    for t in (A, B, aux, C2):
        if t is not None and (t.stride(0) % 8 != 0 or t.data_ptr() % 16 != 0):
            return False
    cmul = 4 if C.dtype == torch.float32 else 8
    return C.stride(0) % cmul == 0 and C.data_ptr() % 16 == 0


def drop_threshold(p):
    """round(256 p) clipped to [0, 255]: the byte threshold of the counter-based dropout masks (csrc/dropout.cuh)."""
    return max(0, min(255, int(round(256.0 * float(p)))))


def attention_desc(qkv, out, lse, T, B, H, dh, sep, dout=None, dqkv=None, delta=None, batch_major=False, drop=None):
    d = AttnDesc()
    if drop is not None:
        d.drop_seed, d.drop_thr = _u32(drop[0]), int(drop[1])
    d.batch_major = int(batch_major)
    d.T, d.B, d.H, d.dh, d.sep = T, B, H, dh, sep
    d.dtype = dtype_code(qkv)
    d.scale = 1.0 / (dh ** 0.5)
    d.qkv, d.ld_qkv = qkv.data_ptr(), qkv.stride(0)
    d.out, d.ld_out = out.data_ptr(), out.stride(0)
    d.lse = lse.data_ptr()
    if dout is not None:
        d.dout, d.ld_dout = dout.data_ptr(), dout.stride(0)
        d.dqkv, d.ld_dqkv = dqkv.data_ptr(), dqkv.stride(0)
        d.delta = delta.data_ptr()
    return d


def tc_attention_ok(qkv, dh, T=None):
    return qkv.dtype == torch.bfloat16 and dh == 128 and qkv.stride(0) % 8 == 0 and qkv.data_ptr() % 16 == 0


@_guarded
def attention_fwd(qkv, out, lse, T, B, H, dh, sep, use_tc=None, batch_major=False, drop=None):
    """drop = (seed, thr): dropout on the attention probabilities (thr 0 / None = off)."""
    d = attention_desc(qkv, out, lse, T, B, H, dh, sep, batch_major=batch_major, drop=drop)
    if use_tc is None:
        use_tc = tc_attention_ok(qkv, dh)
    _call("pfn_attention_fwd_tc" if use_tc else "pfn_attention_fwd_simt", ctypes.byref(d))


@_guarded
def attention_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, dh, sep, use_tc=None, batch_major=False, drop=None,
                  dq_colsum=None, delta_token_major=False):
    """dq_colsum (fp32 [H*dh], tensor-core path only): += column sums of dQ, taken from the staged tiles inside the kernel.
    delta_token_major: `delta` is a [T*B, H] tensor that already holds rowsum(dO * O) (GEMM ROWDOT epilogue)."""
    d = attention_desc(qkv, out, lse, T, B, H, dh, sep, dout, dqkv, delta, batch_major=batch_major, drop=drop)
    if use_tc is None:
        use_tc = tc_attention_ok(qkv, dh)
    if dq_colsum is not None:
        assert use_tc, "dq_colsum is produced by the tensor-core backward only"
        d.dq_colsum = dq_colsum.data_ptr()
    if delta_token_major:
        assert use_tc, "a precomputed token-major delta is consumed by the tensor-core backward only"
        d.delta_token_major = 1
    _call("pfn_attention_bwd_tc" if use_tc else "pfn_attention_bwd_simt", ctypes.byref(d), launches=2)


def attention_ctx_desc(qkv, kv, out, m, n, B, H, dh):
    d = AttnCtxDesc()
    d.m, d.n, d.B, d.H, d.dh = m, n, B, H, dh
    d.dtype = dtype_code(qkv)
    d.scale = 1.0 / (dh ** 0.5)
    d.qkv, d.ld_qkv = qkv.data_ptr(), qkv.stride(0)
    d.kv, d.ld_kv = (kv.data_ptr(), kv.stride(0)) if n > 0 else (None, 0)
    d.out, d.ld_out = out.data_ptr(), out.stride(0)
    return d


def attention_ctx_fwd(qkv, kv, out, m, n, B, H, dh, use_tc=None):
    """out [m*B, H*dh] <- the context attention of the m query rows (packed qkv [m*B, 3*H*dh]) against the n cached training
    rows of the same batch (kv [n*B, 2*H*dh], k | v; unused when n == 0) plus each row's own key."""
    _attention_ctx_fwd(qkv, kv if n > 0 else None, out, m, n, B, H, dh, use_tc)     # an unread kv is not checked


@_guarded
def _attention_ctx_fwd(qkv, kv, out, m, n, B, H, dh, use_tc):
    if qkv.dtype != out.dtype or (n > 0 and kv.dtype != qkv.dtype):
        raise TypeError("attention_ctx_fwd: qkv, kv and out must share one dtype")
    d = attention_ctx_desc(qkv, kv, out, m, n, B, H, dh)
    if use_tc is None:
        use_tc = tc_attention_ok(qkv, dh)
    _call("pfn_attention_ctx_fwd_tc" if use_tc else "pfn_attention_ctx_fwd_simt", ctypes.byref(d))


@_guarded
def embed_fwd(x, y, Wx, bx, wy, by, out, T, B, F, E, sep):
    _call("pfn_embed_fwd", ptr(x), ptr(y), ptr(Wx), ptr(bx), ptr(wy), ptr(by), ptr(out), dtype_code(out), T, B, F, E, sep)


@_guarded
def embed_bwd(dout, x, y, dWx, dbx, dwy, dby, T, B, F, E, sep):
    _call("pfn_embed_bwd", ptr(dout), dtype_code(dout), ptr(x), ptr(y), ptr(dWx), ptr(dbx), ptr(dwy), ptr(dby), T, B, F,
          E, sep, launches=(F + 7) // 8)


@_guarded
def layernorm_fwd(z, gamma, beta, h, mean, rstd, eps=1e-5):
    rows, E = z.shape
    _call("pfn_layernorm_fwd", ptr(z), z.stride(0), ptr(gamma), ptr(beta), ptr(h), h.stride(0), ptr(mean), ptr(rstd),
          rows, E, eps, dtype_code(z))


@_guarded
def layernorm_bwd(dh, z, mean, rstd, gamma, dz, dgamma, dbeta, colsum_out=None):
    rows, E = z.shape
    _call("pfn_layernorm_bwd", ptr(dh), dh.stride(0), ptr(z), z.stride(0), ptr(mean), ptr(rstd), ptr(gamma), ptr(dz),
          dz.stride(0), ptr(dgamma), ptr(dbeta), ptr(colsum_out), rows, E, dtype_code(z))


@_guarded
def colsum(X, out, N=None):
    rows = X.shape[0]
    N = X.shape[1] if N is None else N
    _call("pfn_colsum", ptr(X), X.stride(0), dtype_code(X), ptr(out), rows, N)


@_guarded
def bar_nll_fwd(logits, y, borders, n_bars, full_support, nll, idx, lse, oob_count):
    _call("pfn_bar_nll_fwd", ptr(logits), logits.stride(0), dtype_code(logits), ptr(y), ptr(borders), n_bars,
          int(full_support), ptr(nll), ptr(idx), ptr(lse), ptr(oob_count), logits.shape[0])


@_guarded
def bar_nll_bwd(logits, idx, lse, g, dlogits, n_bars, n_cols_pad=None):
    n_cols_pad = n_bars if n_cols_pad is None else n_cols_pad
    _call("pfn_bar_nll_bwd", ptr(logits), logits.stride(0), dtype_code(logits), ptr(idx), ptr(lse), ptr(g), ptr(dlogits),
          dlogits.stride(0), dtype_code(dlogits), n_bars, n_cols_pad, logits.shape[0])


@_guarded
def bar_bucket_idx(y, borders, n_bars, idx):
    _call("pfn_bar_bucket_idx", ptr(y), ptr(borders), n_bars, ptr(idx), y.numel())


@_guarded
def dropout(x, out, seed, thr, residual=None):
    """out = dropout(x) (+ residual), mask regenerated from (seed, thr); in place when out is x."""
    rows, cols = x.shape
    assert out.shape == x.shape and out.dtype == x.dtype and (residual is None or residual.dtype == x.dtype)
    _call("pfn_dropout", ptr(x), x.stride(0), ptr(residual), residual.stride(0) if residual is not None else 0, ptr(out),
          out.stride(0), rows, cols, dtype_code(x), _u32(seed), int(thr))


@_guarded
def dropout_keep_mask(out, seed, thr):
    """out [rows, cols] uint8 <- keep bits of the site (tests: lets the oracle consume the kernels' mask)."""
    rows, cols = out.shape
    _call("pfn_dropout_keep_mask", ptr(out), rows, cols, _u32(seed), int(thr))


def adam_chunk_elems():
    return int(load().pfn_adam_chunk_elems())


@_guarded
def adam_step(table, chunk_start, n_tensors, n_chunks, lr, beta1, beta2, eps, weight_decay, max_grad_norm, step, norm_sq):
    """Clip (max_grad_norm > 0) + Adam update of every tensor of the device-resident pointer table (optim.FusedClipAdam)."""
    _call("pfn_adam_step", ptr(table), ptr(chunk_start), int(n_tensors), int(n_chunks), float(lr), float(beta1),
          float(beta2), float(eps), float(weight_decay), float(max_grad_norm), int(step), ptr(norm_sq),
          launches=2 if max_grad_norm > 0 else 1)


@_guarded
def gp_sample(x, z, ls, os_, noise, jitter, kernel_type, y, work, info):
    Bn, T, F = x.shape
    _call("pfn_gp_sample", ptr(x), ptr(z), ptr(ls), ptr(os_), ptr(noise), float(jitter), int(kernel_type), ptr(y),
          ptr(work), ptr(info), Bn, T, F)


def _gp_problems(d, B, T, F, ts, kernel_type, hyper):
    """Fills the fields GpFitDesc and GpMcmcDesc share.  hyper = (ls_conc, ls_rate, os_conc, os_rate, noise_conc,
    noise_rate).  The prefix list is kept alive on the descriptor (it is read on the host)."""
    d.B, d.T, d.F = int(B), int(T), int(F)
    d._ts = (c_int * max(len(ts), 1))(*[int(t) for t in ts])
    d.n_ts, d.ts = len(ts), d._ts
    d.kernel_type = int(kernel_type)
    d.ls_conc, d.ls_rate, d.os_conc, d.os_rate, d.noise_conc, d.noise_rate = (float(v) for v in hyper)
    return d


def gp_fit_desc(B, T, F, ts, kernel_type, hyper, noise_lb, noise_init, max_iter, max_eval, ftol, gtol):
    """Descriptor of a pfn_gp_fit call without its device pointers (hyper and ts: see _gp_problems)."""
    d = _gp_problems(GpFitDesc(), B, T, F, ts, kernel_type, hyper)
    d.noise_lb, d.noise_init = float(noise_lb), float(noise_init)
    d.max_iter, d.max_eval, d.ftol, d.gtol = int(max_iter), int(max_eval), float(ftol), float(gtol)
    return d


@_guarded
def gp_fit(x, y, desc, theta, f, iters, nevals, status, theta0=None, grad=None, mean=None, var=None):
    """One launch fits every (prefix in desc.ts, dataset) problem.  x [B,T,F], y [B,T] fp32; outputs indexed by problem
    p = i * B + b: theta / grad [P, F+3], f / mean / var [P] fp64, iters / nevals / status [P] int32."""
    _set_ptrs(desc, x=x, y=y, theta=theta, f=f, iters=iters, nevals=nevals, status=status, theta0=theta0, grad=grad,
              mean=mean, var=var)
    _call("pfn_gp_fit", ctypes.byref(desc))


def gp_mcmc_desc(B, T, F, ts, kernel_type, hyper, num_samples, warmup_steps, seed, max_tree_depth=GP_MCMC_MAX_DEPTH,
                 n_pred=1):
    """Descriptor of a pfn_gp_mcmc call without its device pointers (hyper and ts: see _gp_problems)."""
    d = _gp_problems(GpMcmcDesc(), B, T, F, ts, kernel_type, hyper)
    d.num_samples, d.warmup_steps, d.max_tree_depth = int(num_samples), int(warmup_steps), int(max_tree_depth)
    d.n_pred = int(n_pred)
    d.seed = _u32(seed)
    return d


@_guarded
def gp_mcmc(x, y, desc, samples, step_size, accept, diag, init=None, log_samples=None, mean=None, var=None, potential=None,
            grad=None, trace=None):
    """One launch runs a NUTS chain for every (prefix in desc.ts, dataset) problem.  x [B,T,F], y [B,T] fp32; outputs
    indexed by problem p = i * B + b: samples / log_samples [P, S', F+2], mean / var [P, S', n_pred], potential [P], grad [P, F+2],
    step_size / accept [P] fp64, diag [P, 6] int32 (GP_MCMC_DIAG_NAMES), trace [P, W + S, F+4]; S' = max(num_samples, 1)."""
    _set_ptrs(desc, x=x, y=y, samples=samples, step_size=step_size, accept=accept, diag=diag, init=init,
              log_samples=log_samples, mean=mean, var=var, potential=potential, grad=grad, trace=trace)
    _call("pfn_gp_mcmc", ctypes.byref(desc))


@_guarded
def stroke_geometry(desc, seed, geom, turns, cap_flag):
    """geom [B, C, strokes_max, 4] int32, turns [B, C, strokes_max] fp64 <- the class strokes of B datasets; cap_flag [1]
    int32 is set to 1 (never cleared) when a stroke's rejection loop hits desc.max_iters."""
    _call("pfn_stroke_geometry", ctypes.byref(desc), _u32(seed), geom.shape[0], ptr(geom), ptr(turns), ptr(cap_flag))


@_guarded
def stroke_render(desc, seed, cls, geom, turns, x, normalize):
    """x [T, B, S*S] fp32 <- the images of the class table cls [T, B] int32."""
    T, B = cls.shape
    _call("pfn_stroke_render", ctypes.byref(desc), _u32(seed), ptr(cls), ptr(geom), ptr(turns), ptr(x), T, B,
          int(bool(normalize)))


@_guarded
def stroke_raster(segs, nseg, widths, fill, mask, blurred, S):
    """Oracle hook: mask / blurred [N, S*S] uint8 <- segment sets segs [N, K, 4] int32 (nseg [N], widths [N] int32), ink
    filled with fill [N, S*S] uint8 (None: 128) before the blur."""
    N, K, _ = segs.shape
    _call("pfn_stroke_raster", ptr(segs), ptr(nseg), ptr(widths), ptr(fill), ptr(mask), ptr(blurred), N, K, S)


@_guarded
def omniglot_episodes(desc, seed, bank, alpha_start, x, y, target_y):
    """x [T, B, S*S] fp32, y / target_y [T, B] int64 <- desc.B episodes drawn from bank [n_classes, 20, S, S] uint8
    (alpha_start [n_alpha] int32: first class of every alphabet of the split, Jonas mode only)."""
    _call("pfn_omniglot_episodes", ctypes.byref(desc), _u32(seed), ptr(bank), ptr(alpha_start), ptr(x), ptr(y),
          ptr(target_y))


@_guarded
def bnn_prior(x, y, seed, E, dataset_offset=0, weights=None, x_raw=None, u=None):
    """x [T, B, F] fp32, y [T, B] fp32 <- B datasets of the Bayesian-NN prior with E hidden units.  The oracle hook:
    weights [B, E F + 3 E + 2] fp32, x_raw [T, B, F] fp32 (before the standardisation), u [T, B] fp64 (class uniforms)."""
    T, B, F = x.shape
    _call("pfn_bnn_prior", _u32(seed), int(dataset_offset), B, T, F, int(E), ptr(x), ptr(y), ptr(weights), ptr(x_raw),
          ptr(u))


def bnn_mcmc_desc(N, n, n_test, F, E, num_samples, warmup_steps, seed, max_tree_depth=GP_MCMC_MAX_DEPTH):
    """Descriptor of a pfn_bnn_mcmc call without its device pointers."""
    d = BnnMcmcDesc()
    d.N, d.n, d.n_test, d.F, d.E = int(N), int(n), int(n_test), int(F), int(E)
    d.num_samples, d.warmup_steps, d.max_tree_depth = int(num_samples), int(warmup_steps), int(max_tree_depth)
    d.seed = _u32(seed)
    return d


def bnn_mcmc_workspace(desc):
    """Doubles of global workspace every chain of `desc` needs (0: the sampler state fits in shared memory)."""
    return _workspace("pfn_bnn_mcmc_workspace", desc)


@_guarded
def bnn_mcmc(x_train, y_train, x_test, desc, samples, step_size, accept, diag, init=None, probs=None, obs=None,
             potential=None, grad=None, trace=None, workspace=None):
    """One launch runs a NUTS chain for every dataset.  x_train [N,n,F], y_train [N,n], x_test [N,n_test,F] fp32; outputs
    indexed by dataset: samples [N, S', d], probs [N, S', n_test] fp64, obs [N, S', n_test] fp32 (classes drawn from probs), potential [N], grad [N, d], step_size / accept [N] fp64,
    diag [N, 6] int32 (GP_MCMC_DIAG_NAMES), trace [N, W + S, d + 2]; workspace [N, bnn_mcmc_workspace(desc)] fp64."""
    _set_ptrs(desc, x_train=x_train, y_train=y_train, x_test=x_test, samples=samples, step_size=step_size, accept=accept,
              diag=diag, init=init, probs=probs, obs=obs, potential=potential, grad=grad, trace=trace, workspace=workspace)
    _call("pfn_bnn_mcmc", ctypes.byref(desc))


@_guarded
def knn_cv(x, y, proba, k_best, cv_mean, status):
    """One launch runs the KNN grid-search CV and refit of every problem.  x [n+m, S, F], y [n, S] fp32; outputs
    proba [m, S] fp64, k_best [S] int32, cv_mean [S, min(5, n - 2)] fp64, status [S] int32 (KNN_*)."""
    d = KnnCvDesc()
    rows, d.S, d.F = x.shape
    d.n = y.shape[0]
    d.m = rows - d.n
    _set_ptrs(d, x=x, y=y, proba=proba, k_best=k_best, cv_mean=cv_mean, status=status)
    _call("pfn_knn_cv", ctypes.byref(d))


@_guarded
def ridge_prefix(x, y, target, alpha, pred, sq_err):
    """One launch fits sklearn's Ridge(alpha) to every prefix t = 1 .. T-1 of every dataset.  x [B,T,F], y / target [B,T]
    fp32; outputs pred / sq_err [B,T] fp64 (column 0 NaN)."""
    d = RidgePrefixDesc()
    d.B, d.T, d.F = x.shape
    d.alpha = float(alpha)
    _set_ptrs(d, x=x, y=y, target=target, pred=pred, sq_err=sq_err)
    _call("pfn_ridge_prefix", ctypes.byref(d))


def _exact_gp(x, mode, length_scale, alpha=0.0, **tensors):
    """One pfn_exact_gp call in `mode` on x [B,T,F]; `tensors` sets the descriptor's other pointer fields."""
    d = ExactGpDesc()
    d.B, d.T, d.F = x.shape
    d.mode, d.length_scale, d.alpha = mode, float(length_scale), float(alpha)
    _call("pfn_exact_gp", ctypes.byref(_set_ptrs(d, x=x, **tensors)))


@_guarded
def exact_gp_evaluate(x, y, length_scale, alpha, mean, var, status):
    """The RBF exact GP's predictive of row t given rows < t, every t = 1 .. T-1 and dataset, from one factor per dataset.
    x [B,T,F], y [B,T] fp32; outputs mean / var [B,T] fp64 (column 0 NaN), status [B] int32 (0 or the failing prefix)."""
    _exact_gp(x, EXACT_GP_EVALUATE, length_scale, alpha, y=y, mean=mean, var=var, status=status)


@_guarded
def exact_gp_sample(x, z, length_scale, sample, rank, factor=None, perm=None):
    """sample [B,T] fp32 = P L z[:, :r] with P L L^T P^T = RBF(x, x) (pivoted Cholesky to the numerical rank r); rank [B]
    int32; optional factor [B,T,T] fp64 (P L) and perm [B,T] int32 (pivot order)."""
    _exact_gp(x, EXACT_GP_SAMPLE, length_scale, z=z, sample=sample, rank=rank, factor=factor, perm=perm)


# ------------------------------------------------------------------------------------------------
# what the two NUTS samplers (gp_mcmc, bnn_mcmc) share on the host
# ------------------------------------------------------------------------------------------------
def mcmc_outputs(n, d, num_samples, warmup_steps, trace, device):
    """The per-chain outputs of n chains over d coordinates: samples [n, S', d], potential [n], grad [n, d], step_size /
    accept [n] fp64, diag [n, 6] int32 and, when `trace`, trace [n, W + S, d + 2]; S' = max(num_samples, 1)."""
    f64 = dict(dtype=torch.float64, device=device)
    out = {"samples": torch.empty(n, max(int(num_samples), 1), d, **f64), "potential": torch.empty(n, **f64),
           "grad": torch.empty(n, d, **f64), "step_size": torch.empty(n, **f64), "accept": torch.empty(n, **f64),
           "diag": torch.empty(n, len(GP_MCMC_DIAG_NAMES), dtype=torch.int32, device=device)}
    if trace:
        out["trace"] = torch.empty(n, int(warmup_steps) + int(num_samples), d + 2, **f64)
    return out


def mcmc_trouble(diag):
    """(divergent sampling iterations, iterations that hit the tree-depth cap) summed over the chains of diag [..., 6]."""
    col = GP_MCMC_DIAG_NAMES.index
    return int(diag[..., col("div_sampling")].sum()), int(diag[..., col("max_depth_hits")].sum())


def _conv_desc(N, S, C_in, dtype, **tensors):
    """Descriptor of one 3x3 layer of the conv encoder (include/pfn_b200.h, pfn_conv_desc); S is the layer's input side,
    `tensors` sets its pointer fields (x, w, bias, g, y, dw, db, workspace; the others stay NULL)."""
    d = ConvDesc()
    d.N, d.S, d.C_in, d.dtype = N, S, C_in, dtype_code(dtype) if torch.is_tensor(dtype) else dtype
    return _set_ptrs(d, **tensors)


@_guarded
def conv_fwd(x, w, bias, y, N, S, C_in):
    """y [N, S-2, S-2, 64] = relu(conv3x3(x) + bias); y's dtype is the activation dtype."""
    _call("pfn_conv_fwd", ctypes.byref(_conv_desc(N, S, C_in, y, x=x, w=w, bias=bias, y=y)))


@_guarded
def conv_dgrad(g, w, x, out, N, S):
    """out (padded, side S + 4) interior = (input gradient of the 64 -> 64 layer with input x) * [x > 0]."""
    _call("pfn_conv_dgrad", ctypes.byref(_conv_desc(N, S, CONV_CH, out, x=x, w=w, g=g, y=out)))


def conv_wgrad_workspace(N, S, C_in):
    return _workspace("pfn_conv_wgrad_workspace", _conv_desc(N, S, C_in, F32))


@_guarded
def conv_wgrad(g, x, dw, db, N, S, C_in):
    """dw [64, C_in, 3, 3], db [64] fp32 (overwritten) of the layer with input x and padded output gradient g."""
    ws = torch.empty(conv_wgrad_workspace(N, S, C_in), device=g.device, dtype=torch.float32)
    _call("pfn_conv_wgrad", ctypes.byref(_conv_desc(N, S, C_in, g, x=x, g=g, dw=dw, db=db, workspace=ws)), launches=2)


@_guarded
def conv_mean_fwd(y, feat, N, s):
    _call("pfn_conv_mean_fwd", ptr(y), N, s, dtype_code(y), ptr(feat))


@_guarded
def conv_mean_bwd(dfeat, y, g, N, s):
    _call("pfn_conv_mean_bwd", ptr(dfeat), ptr(y), N, s, dtype_code(y), ptr(g))


# ------------------------------------------------------------------------------------------------
# learned-temperature decoder heads (csrc/scaled_head.cu)
# ------------------------------------------------------------------------------------------------
@_guarded
def scaled_head_fwd(zz, n_out, out, temp):
    """out [rows, n_out] = zz[:, :n_out] / temp, temp [rows] = softmax(zz[:, n_out:n_out + 10]) . c; zz, out, temp fp32."""
    _call("pfn_scaled_head_fwd", ptr(zz), zz.stride(0), int(n_out), ptr(out), out.stride(0), ptr(temp), zz.shape[0])


@_guarded
def scaled_head_bwd(g, zz, temp, n_out, dzz, n_cols_pad=None):
    """dzz [rows, n_cols_pad] (activation dtype) <- g [rows, n_out] fp32, the forward's zz and temp."""
    n_cols_pad = n_out + HEAD_TEMPS if n_cols_pad is None else n_cols_pad
    _call("pfn_scaled_head_bwd", ptr(g), g.stride(0), ptr(zz), zz.stride(0), ptr(temp), int(n_out), ptr(dzz),
          dzz.stride(0), dtype_code(dzz), int(n_cols_pad), g.shape[0])


@_guarded
def fixed_scaled_head_fwd(z, n_out, T, out, S):
    """out [rows, n_out] = z[:, :n_out] / S with S [1] = sum(T), all fp32."""
    _call("pfn_fixed_scaled_head_fwd", ptr(z), z.stride(0), int(n_out), ptr(T), T.numel(), ptr(out), out.stride(0),
          ptr(S), z.shape[0])


@_guarded
def fixed_scaled_head_bwd(g, z, S, n_out, dz, dT, n_cols_pad=None, row_dot=None):
    """dz [rows, n_cols_pad] (activation dtype) = g / S; every dT [n_t] = -sum(g z) / S^2 (fp32)."""
    rows = g.shape[0]
    if row_dot is None:
        row_dot = torch.empty(rows, device=g.device, dtype=torch.float32)
    n_cols_pad = n_out if n_cols_pad is None else n_cols_pad
    _call("pfn_fixed_scaled_head_bwd", ptr(g), g.stride(0), ptr(z), z.stride(0), ptr(S), int(n_out), ptr(dz),
          dz.stride(0), dtype_code(dz), int(n_cols_pad), ptr(row_dot), ptr(dT), dT.numel(), rows,
          launches=2 if rows else 1)
