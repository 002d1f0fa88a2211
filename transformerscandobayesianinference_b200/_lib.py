"""ctypes binding of libpfn_b200.so (the C ABI declared in include/pfn_b200.h).

There is deliberately no fallback: if the shared object is missing or a call fails, a RuntimeError with the
library's own message is raised.  Tensors are passed as raw device pointers on torch's current CUDA stream.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# PFN_B200_LIB points at another build of the same library (A/B measurements of kernel variants); default: the in-tree build
LIB_PATH = os.environ.get("PFN_B200_LIB") or os.path.join(_HERE, "libpfn_b200.so")

F32, BF16 = 0, 1
EPI_NONE, EPI_GELU, EPI_GELU_BWD, EPI_ROWDOT, EPI_MUL = 0, 1, 2, 3, 4
KERNEL_RBF, KERNEL_MATERN12, KERNEL_MATERN32, KERNEL_MATERN52 = 0, 1, 2, 3

c_int, c_float, c_void_p = ctypes.c_int, ctypes.c_float, ctypes.c_void_p


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


c_double = ctypes.c_double


class GpFitDesc(ctypes.Structure):
    _fields_ = [
        ("B", c_int), ("T", c_int), ("F", c_int),
        ("x", c_void_p), ("y", c_void_p),
        ("n_ts", c_int), ("ts", ctypes.POINTER(c_int)),
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
        ("n_ts", c_int), ("ts", ctypes.POINTER(c_int)),
        ("kernel_type", c_int),
        ("ls_conc", c_double), ("ls_rate", c_double), ("os_conc", c_double), ("os_rate", c_double),
        ("noise_conc", c_double), ("noise_rate", c_double),
        ("num_samples", c_int), ("warmup_steps", c_int), ("max_tree_depth", c_int), ("n_pred", c_int),
        ("seed", ctypes.c_uint32),
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
        ("seed", ctypes.c_uint32),
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
        ("drop_seed", ctypes.c_uint32), ("drop_thr", c_int),
        ("dq_colsum", c_void_p), ("delta_token_major", c_int),
    ]


EXPORTED_SYMBOLS = [
    "pfn_last_error", "pfn_version", "pfn_num_sms",
    "pfn_gemm_bf16_tc", "pfn_gemm_simt",
    "pfn_attention_fwd_simt", "pfn_attention_bwd_simt", "pfn_attention_fwd_tc", "pfn_attention_bwd_tc",
    "pfn_embed_fwd", "pfn_embed_bwd",
    "pfn_layernorm_fwd", "pfn_layernorm_bwd", "pfn_colsum",
    "pfn_bar_nll_fwd", "pfn_bar_nll_bwd", "pfn_bar_bucket_idx",
    "pfn_gp_sample", "pfn_gp_fit", "pfn_gp_mcmc",
    "pfn_dropout", "pfn_dropout_keep_mask",
    "pfn_adam_step", "pfn_adam_chunk_elems",
    "pfn_stroke_geometry", "pfn_stroke_render", "pfn_stroke_raster",
    "pfn_omniglot_episodes",
    "pfn_bnn_prior", "pfn_bnn_mcmc_workspace", "pfn_bnn_mcmc",
    "pfn_knn_cv",
]

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


def _count(n=1):
    global _launches
    _launches += n


def load():
    """Load (once) and return the ctypes handle.  Raises if the library has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU / PyTorch fallback for the PFN hot path)")
    lib = ctypes.CDLL(LIB_PATH)
    lib.pfn_last_error.restype = ctypes.c_char_p
    for name in EXPORTED_SYMBOLS:
        if not hasattr(lib, name):
            raise RuntimeError(f"libpfn_b200.so does not export {name}")
        if name != "pfn_last_error":
            getattr(lib, name).restype = c_int
    lib.pfn_gemm_bf16_tc.argtypes = [ctypes.POINTER(GemmDesc), c_void_p]
    lib.pfn_gemm_simt.argtypes = [ctypes.POINTER(GemmDesc), c_void_p]
    for n in ("pfn_attention_fwd_simt", "pfn_attention_bwd_simt", "pfn_attention_fwd_tc", "pfn_attention_bwd_tc"):
        getattr(lib, n).argtypes = [ctypes.POINTER(AttnDesc), c_void_p]
    lib.pfn_embed_fwd.argtypes = [c_void_p] * 7 + [c_int] * 6 + [c_void_p]
    lib.pfn_embed_bwd.argtypes = [c_void_p, c_int] + [c_void_p] * 6 + [c_int] * 5 + [c_void_p]
    lib.pfn_layernorm_fwd.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                      c_int, c_int, c_float, c_int, c_void_p]
    lib.pfn_layernorm_bwd.argtypes = [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                      c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]
    lib.pfn_colsum.argtypes = [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p]
    lib.pfn_bar_nll_fwd.argtypes = [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_int, c_void_p]
    lib.pfn_bar_nll_bwd.argtypes = [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                    c_int, c_int, c_int, c_void_p]
    lib.pfn_bar_bucket_idx.argtypes = [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p]
    lib.pfn_gp_sample.argtypes = [c_void_p] * 5 + [c_float, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                  c_void_p]
    lib.pfn_gp_fit.argtypes = [ctypes.POINTER(GpFitDesc), c_void_p]
    lib.pfn_gp_mcmc.argtypes = [ctypes.POINTER(GpMcmcDesc), c_void_p]
    lib.pfn_dropout.argtypes = [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, ctypes.c_uint32, c_int,
                                c_void_p]
    lib.pfn_dropout_keep_mask.argtypes = [c_void_p, c_int, c_int, ctypes.c_uint32, c_int, c_void_p]
    lib.pfn_stroke_geometry.argtypes = [ctypes.POINTER(StrokeDesc), ctypes.c_uint32, c_int, c_void_p, c_void_p, c_void_p,
                                        c_void_p]
    lib.pfn_stroke_render.argtypes = [ctypes.POINTER(StrokeDesc), ctypes.c_uint32, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_int, c_int, c_int, c_void_p]
    lib.pfn_stroke_raster.argtypes = [c_void_p] * 6 + [c_int, c_int, c_int, c_void_p]
    lib.pfn_omniglot_episodes.argtypes = [ctypes.POINTER(OmniglotDesc), ctypes.c_uint32] + [c_void_p] * 6
    lib.pfn_bnn_prior.argtypes = [ctypes.c_uint32] + [c_int] * 5 + [c_void_p] * 6
    lib.pfn_bnn_mcmc_workspace.argtypes = [ctypes.POINTER(BnnMcmcDesc)]
    lib.pfn_bnn_mcmc.argtypes = [ctypes.POINTER(BnnMcmcDesc), c_void_p]
    lib.pfn_knn_cv.argtypes = [ctypes.POINTER(KnnCvDesc), c_void_p]
    _lib = lib
    return lib


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


def _guarded(fn):
    """Run the wrapped library call with the device of its first tensor argument as the current device (so that
    `stream_ptr()`, `num_sms()` and the launch itself all refer to the device that owns the data)."""
    import functools

    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        dev = None
        for a in args:
            if torch.is_tensor(a) and a.is_cuda:
                dev = a.device
                break
        if dev is None:
            return fn(*args, **kwargs)
        with on_device(dev):
            return fn(*args, **kwargs)
    return wrapper


# ------------------------------------------------------------------------------------------------
# thin wrappers
# ------------------------------------------------------------------------------------------------
@_guarded
def gemm(A, B, C, *, a_mn_major=False, b_mn_major=False, bias=None, aux=None, C2=None, epilogue=EPI_NONE,
         accumulate=False, k_splits=1, M=None, N=None, K=None, use_tc=None, rowdot=None, c2_gelu_grad=False):
    """C[M,N] (+)= epi(A . B^T-ish + bias) (+ aux).  Operands are 2-D row-major tensors (stride(1) == 1)."""
    lib = load()
    require_cuda(A, B, C, bias, aux, C2)
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
        require_cuda(rowdot[0])
        d.rowdot_out, d.rowdot_width = rowdot[0].data_ptr(), int(rowdot[1])
    if use_tc is None:
        use_tc = tc_gemm_ok(A, B, C, aux, C2)
    _count()
    if use_tc:
        if PROFILE_GEMM is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            check(lib.pfn_gemm_bf16_tc(ctypes.byref(d), stream_ptr()), "pfn_gemm_bf16_tc")
            e1.record()
            esz = 4 if C.dtype == torch.float32 else 2
            nbytes = 2.0 * (M * K + N * K) + esz * M * N * (2 if C2 is not None else 1) + (2.0 * M * N if aux is not None else 0.0)
            PROFILE_GEMM.append((2.0 * M * N * K, e0, e1, nbytes))
        else:
            check(lib.pfn_gemm_bf16_tc(ctypes.byref(d), stream_ptr()), "pfn_gemm_bf16_tc")
    else:
        check(lib.pfn_gemm_simt(ctypes.byref(d), stream_ptr()), "pfn_gemm_simt")


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
        d.drop_seed, d.drop_thr = int(drop[0]) & 0xFFFFFFFF, int(drop[1])
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
    _count(1)
    lib = load()
    require_cuda(qkv, out, lse)
    d = attention_desc(qkv, out, lse, T, B, H, dh, sep, batch_major=batch_major, drop=drop)
    if use_tc is None:
        use_tc = tc_attention_ok(qkv, dh)
    fn = lib.pfn_attention_fwd_tc if use_tc else lib.pfn_attention_fwd_simt
    check(fn(ctypes.byref(d), stream_ptr()), "pfn_attention_fwd")


@_guarded
def attention_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, dh, sep, use_tc=None, batch_major=False, drop=None,
                  dq_colsum=None, delta_token_major=False):
    """dq_colsum (fp32 [H*dh], tensor-core path only): += column sums of dQ, taken from the staged tiles inside the kernel.
    delta_token_major: `delta` is a [T*B, H] tensor that already holds rowsum(dO * O) (GEMM ROWDOT epilogue)."""
    _count(2)
    lib = load()
    require_cuda(qkv, out, lse, dout, dqkv, delta, dq_colsum)
    d = attention_desc(qkv, out, lse, T, B, H, dh, sep, dout, dqkv, delta, batch_major=batch_major, drop=drop)
    if use_tc is None:
        use_tc = tc_attention_ok(qkv, dh)
    if dq_colsum is not None:
        assert use_tc, "dq_colsum is produced by the tensor-core backward only"
        d.dq_colsum = dq_colsum.data_ptr()
    if delta_token_major:
        assert use_tc, "a precomputed token-major delta is consumed by the tensor-core backward only"
        d.delta_token_major = 1
    fn = lib.pfn_attention_bwd_tc if use_tc else lib.pfn_attention_bwd_simt
    check(fn(ctypes.byref(d), stream_ptr()), "pfn_attention_bwd")


@_guarded
def embed_fwd(x, y, Wx, bx, wy, by, out, T, B, F, E, sep):
    _count(1)
    require_cuda(x, y, Wx, bx, wy, by, out)
    check(load().pfn_embed_fwd(ptr(x), ptr(y), ptr(Wx), ptr(bx), ptr(wy), ptr(by), ptr(out), dtype_code(out), T, B, F,
                               E, sep, stream_ptr()), "pfn_embed_fwd")


@_guarded
def embed_bwd(dout, x, y, dWx, dbx, dwy, dby, T, B, F, E, sep):
    _count((F + 7) // 8)
    require_cuda(dout, x, y, dWx, dbx, dwy, dby)
    check(load().pfn_embed_bwd(ptr(dout), dtype_code(dout), ptr(x), ptr(y), ptr(dWx), ptr(dbx), ptr(dwy), ptr(dby), T,
                               B, F, E, sep, stream_ptr()), "pfn_embed_bwd")


@_guarded
def layernorm_fwd(z, gamma, beta, h, mean, rstd, eps=1e-5):
    _count(1)
    require_cuda(z, gamma, beta, h, mean, rstd)
    rows, E = z.shape
    check(load().pfn_layernorm_fwd(ptr(z), z.stride(0), ptr(gamma), ptr(beta), ptr(h), h.stride(0), ptr(mean),
                                   ptr(rstd), rows, E, eps, dtype_code(z), stream_ptr()), "pfn_layernorm_fwd")


@_guarded
def layernorm_bwd(dh, z, mean, rstd, gamma, dz, dgamma, dbeta, colsum_out=None):
    _count(1)
    require_cuda(dh, z, mean, rstd, gamma, dz, dgamma, dbeta, colsum_out)
    rows, E = z.shape
    check(load().pfn_layernorm_bwd(ptr(dh), dh.stride(0), ptr(z), z.stride(0), ptr(mean), ptr(rstd), ptr(gamma),
                                   ptr(dz), dz.stride(0), ptr(dgamma), ptr(dbeta), ptr(colsum_out), rows, E,
                                   dtype_code(z), stream_ptr()), "pfn_layernorm_bwd")


@_guarded
def colsum(X, out, N=None):
    _count(1)
    require_cuda(X, out)
    rows = X.shape[0]
    N = X.shape[1] if N is None else N
    check(load().pfn_colsum(ptr(X), X.stride(0), dtype_code(X), ptr(out), rows, N, stream_ptr()), "pfn_colsum")


@_guarded
def bar_nll_fwd(logits, y, borders, n_bars, full_support, nll, idx, lse, oob_count):
    _count(1)
    require_cuda(logits, y, borders, nll, idx, lse, oob_count)
    rows = logits.shape[0]
    check(load().pfn_bar_nll_fwd(ptr(logits), logits.stride(0), dtype_code(logits), ptr(y), ptr(borders), n_bars,
                                 int(full_support), ptr(nll), ptr(idx), ptr(lse), ptr(oob_count), rows, stream_ptr()),
          "pfn_bar_nll_fwd")


@_guarded
def bar_nll_bwd(logits, idx, lse, g, dlogits, n_bars, n_cols_pad=None):
    _count(1)
    require_cuda(logits, idx, lse, g, dlogits)
    rows = logits.shape[0]
    n_cols_pad = n_bars if n_cols_pad is None else n_cols_pad
    check(load().pfn_bar_nll_bwd(ptr(logits), logits.stride(0), dtype_code(logits), ptr(idx), ptr(lse), ptr(g),
                                 ptr(dlogits), dlogits.stride(0), dtype_code(dlogits), n_bars, n_cols_pad, rows,
                                 stream_ptr()), "pfn_bar_nll_bwd")


@_guarded
def bar_bucket_idx(y, borders, n_bars, idx):
    _count(1)
    require_cuda(y, borders, idx)
    check(load().pfn_bar_bucket_idx(ptr(y), ptr(borders), n_bars, ptr(idx), y.numel(), stream_ptr()),
          "pfn_bar_bucket_idx")


@_guarded
def dropout(x, out, seed, thr, residual=None):
    """out = dropout(x) (+ residual), mask regenerated from (seed, thr); in place when out is x."""
    _count(1)
    require_cuda(x, out, residual)
    rows, cols = x.shape
    assert out.shape == x.shape and out.dtype == x.dtype and (residual is None or residual.dtype == x.dtype)
    check(load().pfn_dropout(ptr(x), x.stride(0), ptr(residual), residual.stride(0) if residual is not None else 0, ptr(out),
                             out.stride(0), rows, cols, dtype_code(x), int(seed) & 0xFFFFFFFF, int(thr), stream_ptr()), "pfn_dropout")


@_guarded
def dropout_keep_mask(out, seed, thr):
    """out [rows, cols] uint8 <- keep bits of the site (tests: lets the oracle consume the kernels' mask)."""
    _count(1)
    require_cuda(out)
    rows, cols = out.shape
    check(load().pfn_dropout_keep_mask(ptr(out), rows, cols, int(seed) & 0xFFFFFFFF, int(thr), stream_ptr()), "pfn_dropout_keep_mask")


def adam_chunk_elems():
    return int(load().pfn_adam_chunk_elems())


@_guarded
def adam_step(table, chunk_start, n_tensors, n_chunks, lr, beta1, beta2, eps, weight_decay, max_grad_norm, step, norm_sq):
    """Clip (max_grad_norm > 0) + Adam update of every tensor of the device-resident pointer table (optim.FusedClipAdam)."""
    _count(2 if max_grad_norm > 0 else 1)
    require_cuda(table, chunk_start, norm_sq)
    c_float = ctypes.c_float
    fn = load().pfn_adam_step
    fn.argtypes = [c_void_p, c_void_p, c_int, c_int, c_float, c_float, c_float, c_float, c_float, c_float, c_int, c_void_p,
                   c_void_p]
    check(fn(ptr(table), ptr(chunk_start), int(n_tensors), int(n_chunks), float(lr), float(beta1), float(beta2), float(eps),
             float(weight_decay), float(max_grad_norm), int(step), ptr(norm_sq), stream_ptr()), "pfn_adam_step")


@_guarded
def gp_sample(x, z, ls, os_, noise, jitter, kernel_type, y, work, info):
    _count(1)
    require_cuda(x, z, ls, os_, noise, y, work, info)
    Bn, T, F = x.shape
    check(load().pfn_gp_sample(ptr(x), ptr(z), ptr(ls), ptr(os_), ptr(noise), float(jitter), int(kernel_type), ptr(y),
                               ptr(work), ptr(info), Bn, T, F, stream_ptr()), "pfn_gp_sample")


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
    _count(1)
    require_cuda(x, y, theta, f, iters, nevals, status, theta0, grad, mean, var)
    desc.x, desc.y = x.data_ptr(), y.data_ptr()
    desc.theta, desc.f = theta.data_ptr(), f.data_ptr()
    desc.iters, desc.nevals, desc.status = iters.data_ptr(), nevals.data_ptr(), status.data_ptr()
    desc.theta0, desc.grad, desc.mean, desc.var = ptr(theta0), ptr(grad), ptr(mean), ptr(var)
    check(load().pfn_gp_fit(ctypes.byref(desc), stream_ptr()), "pfn_gp_fit")


def gp_mcmc_desc(B, T, F, ts, kernel_type, hyper, num_samples, warmup_steps, seed, max_tree_depth=GP_MCMC_MAX_DEPTH,
                 n_pred=1):
    """Descriptor of a pfn_gp_mcmc call without its device pointers (hyper and ts: see _gp_problems)."""
    d = _gp_problems(GpMcmcDesc(), B, T, F, ts, kernel_type, hyper)
    d.num_samples, d.warmup_steps, d.max_tree_depth = int(num_samples), int(warmup_steps), int(max_tree_depth)
    d.n_pred = int(n_pred)
    d.seed = int(seed) & 0xFFFFFFFF
    return d


@_guarded
def gp_mcmc(x, y, desc, samples, step_size, accept, diag, init=None, log_samples=None, mean=None, var=None, potential=None,
            grad=None, trace=None):
    """One launch runs a NUTS chain for every (prefix in desc.ts, dataset) problem.  x [B,T,F], y [B,T] fp32; outputs
    indexed by problem p = i * B + b: samples / log_samples [P, S', F+2], mean / var [P, S', n_pred], potential [P], grad [P, F+2],
    step_size / accept [P] fp64, diag [P, 6] int32 (GP_MCMC_DIAG_NAMES), trace [P, W + S, F+4]; S' = max(num_samples, 1)."""
    _count(1)
    require_cuda(x, y, samples, step_size, accept, diag, init, log_samples, mean, var, potential, grad, trace)
    desc.x, desc.y = x.data_ptr(), y.data_ptr()
    desc.samples, desc.step_size, desc.accept, desc.diag = (samples.data_ptr(), step_size.data_ptr(), accept.data_ptr(),
                                                            diag.data_ptr())
    desc.init, desc.log_samples, desc.mean, desc.var = ptr(init), ptr(log_samples), ptr(mean), ptr(var)
    desc.potential, desc.grad, desc.trace = ptr(potential), ptr(grad), ptr(trace)
    check(load().pfn_gp_mcmc(ctypes.byref(desc), stream_ptr()), "pfn_gp_mcmc")


@_guarded
def stroke_geometry(desc, seed, geom, turns, cap_flag):
    """geom [B, C, strokes_max, 4] int32, turns [B, C, strokes_max] fp64 <- the class strokes of B datasets; cap_flag [1]
    int32 is set to 1 (never cleared) when a stroke's rejection loop hits desc.max_iters."""
    _count(1)
    require_cuda(geom, turns, cap_flag)
    check(load().pfn_stroke_geometry(ctypes.byref(desc), int(seed) & 0xFFFFFFFF, geom.shape[0], ptr(geom), ptr(turns),
                                     ptr(cap_flag), stream_ptr()), "pfn_stroke_geometry")


@_guarded
def stroke_render(desc, seed, cls, geom, turns, x, normalize):
    """x [T, B, S*S] fp32 <- the images of the class table cls [T, B] int32."""
    _count(1)
    require_cuda(cls, geom, turns, x)
    T, B = cls.shape
    check(load().pfn_stroke_render(ctypes.byref(desc), int(seed) & 0xFFFFFFFF, ptr(cls), ptr(geom), ptr(turns), ptr(x), T, B,
                                   int(bool(normalize)), stream_ptr()), "pfn_stroke_render")


@_guarded
def stroke_raster(segs, nseg, widths, fill, mask, blurred, S):
    """Oracle hook: mask / blurred [N, S*S] uint8 <- segment sets segs [N, K, 4] int32 (nseg [N], widths [N] int32), ink
    filled with fill [N, S*S] uint8 (None: 128) before the blur."""
    _count(1)
    require_cuda(segs, nseg, widths, fill, mask, blurred)
    N, K, _ = segs.shape
    check(load().pfn_stroke_raster(ptr(segs), ptr(nseg), ptr(widths), ptr(fill), ptr(mask), ptr(blurred), N, K, S,
                                   stream_ptr()), "pfn_stroke_raster")


@_guarded
def omniglot_episodes(desc, seed, bank, alpha_start, x, y, target_y):
    """x [T, B, S*S] fp32, y / target_y [T, B] int64 <- desc.B episodes drawn from bank [n_classes, 20, S, S] uint8
    (alpha_start [n_alpha] int32: first class of every alphabet of the split, Jonas mode only)."""
    _count(1)
    require_cuda(bank, alpha_start, x, y, target_y)
    check(load().pfn_omniglot_episodes(ctypes.byref(desc), int(seed) & 0xFFFFFFFF, ptr(bank), ptr(alpha_start), ptr(x), ptr(y),
                                       ptr(target_y), stream_ptr()), "pfn_omniglot_episodes")


@_guarded
def bnn_prior(x, y, seed, E, dataset_offset=0, weights=None, x_raw=None, u=None):
    """x [T, B, F] fp32, y [T, B] fp32 <- B datasets of the Bayesian-NN prior with E hidden units.  The oracle hook:
    weights [B, E F + 3 E + 2] fp32, x_raw [T, B, F] fp32 (before the standardisation), u [T, B] fp64 (class uniforms)."""
    _count(1)
    require_cuda(x, y, weights, x_raw, u)
    T, B, F = x.shape
    check(load().pfn_bnn_prior(int(seed) & 0xFFFFFFFF, int(dataset_offset), B, T, F, int(E), ptr(x), ptr(y), ptr(weights),
                               ptr(x_raw), ptr(u), stream_ptr()), "pfn_bnn_prior")


def bnn_mcmc_desc(N, n, n_test, F, E, num_samples, warmup_steps, seed, max_tree_depth=GP_MCMC_MAX_DEPTH):
    """Descriptor of a pfn_bnn_mcmc call without its device pointers."""
    d = BnnMcmcDesc()
    d.N, d.n, d.n_test, d.F, d.E = int(N), int(n), int(n_test), int(F), int(E)
    d.num_samples, d.warmup_steps, d.max_tree_depth = int(num_samples), int(warmup_steps), int(max_tree_depth)
    d.seed = int(seed) & 0xFFFFFFFF
    return d


def bnn_mcmc_workspace(desc):
    """Doubles of global workspace every chain of `desc` needs (0: the sampler state fits in shared memory)."""
    w = int(load().pfn_bnn_mcmc_workspace(ctypes.byref(desc)))
    if w < 0:
        check(1, "pfn_bnn_mcmc_workspace")
    return w


@_guarded
def bnn_mcmc(x_train, y_train, x_test, desc, samples, step_size, accept, diag, init=None, probs=None, obs=None,
             potential=None, grad=None, trace=None, workspace=None):
    """One launch runs a NUTS chain for every dataset.  x_train [N,n,F], y_train [N,n], x_test [N,n_test,F] fp32; outputs
    indexed by dataset: samples [N, S', d], probs [N, S', n_test] fp64, obs [N, S', n_test] fp32 (classes drawn from probs), potential [N], grad [N, d], step_size / accept [N] fp64,
    diag [N, 6] int32 (GP_MCMC_DIAG_NAMES), trace [N, W + S, d + 2]; workspace [N, bnn_mcmc_workspace(desc)] fp64."""
    _count(1)
    require_cuda(x_train, y_train, x_test, samples, step_size, accept, diag, init, probs, obs, potential, grad, trace, workspace)
    desc.x_train, desc.y_train, desc.x_test = x_train.data_ptr(), y_train.data_ptr(), ptr(x_test)
    desc.init = ptr(init)
    desc.samples, desc.step_size, desc.accept, desc.diag = (samples.data_ptr(), step_size.data_ptr(), accept.data_ptr(),
                                                            diag.data_ptr())
    desc.probs, desc.obs, desc.potential, desc.grad = ptr(probs), ptr(obs), ptr(potential), ptr(grad)
    desc.trace, desc.workspace = ptr(trace), ptr(workspace)
    check(load().pfn_bnn_mcmc(ctypes.byref(desc), stream_ptr()), "pfn_bnn_mcmc")


@_guarded
def knn_cv(x, y, proba, k_best, cv_mean, status):
    """One launch runs the KNN grid-search CV and refit of every problem.  x [n+m, S, F], y [n, S] fp32; outputs
    proba [m, S] fp64, k_best [S] int32, cv_mean [S, min(5, n - 2)] fp64, status [S] int32 (KNN_*)."""
    _count(1)
    require_cuda(x, y, proba, k_best, cv_mean, status)
    d = KnnCvDesc()
    rows, d.S, d.F = x.shape
    d.n = y.shape[0]
    d.m = rows - d.n
    d.x, d.y = x.data_ptr(), y.data_ptr()
    d.proba, d.k_best, d.cv_mean, d.status = proba.data_ptr(), k_best.data_ptr(), cv_mean.data_ptr(), status.data_ptr()
    check(load().pfn_knn_cv(ctypes.byref(d), stream_ptr()), "pfn_knn_cv")


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
