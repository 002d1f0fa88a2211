"""Every public wrapper of the ctypes binding (_lib.py) on the host, against a recording fake of the library.

For each call the log holds the entry points invoked, in order, with every argument decoded (a pointer as the name of
the argument tensor it points into plus a byte offset, a descriptor field by field, a `POINTER(c_int)` array as its
values), the launches the call adds to `launch_count()`, and which of its tensor arguments it hands to `require_cuda`.
tests/golden/lib_calls.json holds that log; `python tests/test_lib_calls_host.py` rewrites it.  A CPU tensor in any
tensor argument must be rejected before the library is called or a launch is counted."""
import ctypes
import inspect
import json
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from transformerscandobayesianinference_b200 import _lib as L  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "lib_calls.json")
STREAM = object()                                   # what the patched stream_ptr() returns
QUERIES = {"pfn_bnn_mcmc_workspace": 40, "pfn_conv_wgrad_workspace": 24, "pfn_adam_chunk_elems": 4096}
NOT_CALLED = {"pfn_last_error", "pfn_version", "pfn_num_sms"}
BF16, F32, F64, I32, I64, U8 = torch.bfloat16, torch.float32, torch.float64, torch.int32, torch.int64, torch.uint8


def t(*shape, dtype=F32):
    return torch.zeros(shape, dtype=dtype)


def _gp_hyper():
    return (1.5, 2.0, 3.0, 4.0, 5.0, 6.0)


def _stroke_desc():
    d = L.StrokeDesc()
    d.S, d.C, d.strokes_min, d.strokes_max, d.max_iters = 28, 3, 1, 4, 100
    return d


def _omniglot_desc():
    d = L.OmniglotDesc()
    d.S, d.n_classes, d.B, d.n_way, d.k_shot, d.T = 28, 10, 2, 3, 1, 6
    return d


def _attn(T=8, B=2, H=2, dh=4, dtype=BF16):
    return t(T * B, 3 * H * dh, dtype=dtype), t(T * B, H * dh, dtype=dtype), t(B * H * T)


# (case, wrapper, builder of (args, kwargs)); every builder makes fresh tensors and descriptors
CASES = [
    ("gemm_tc", "gemm", lambda: ((t(16, 32, dtype=BF16), t(24, 32, dtype=BF16), t(16, 24)),
                                 dict(bias=t(24), use_tc=True))),
    ("gemm_simt_gelu", "gemm", lambda: ((t(32, 16), t(32, 24), t(16, 24)),
                                        dict(a_mn_major=True, b_mn_major=True, aux=t(16, 24), C2=t(16, 24),
                                             epilogue=L.EPI_GELU, accumulate=True, k_splits=2, use_tc=False,
                                             c2_gelu_grad=True))),
    ("gemm_rowdot", "gemm", lambda: ((t(16, 32, dtype=BF16), t(24, 32, dtype=BF16), t(16, 24, dtype=BF16)),
                                     dict(epilogue=L.EPI_ROWDOT, rowdot=(t(16, 3), 8), M=16, N=24, K=32, use_tc=True))),
    ("attention_fwd_tc", "attention_fwd", lambda: ((*_attn(), 8, 2, 2, 4, 5), dict(use_tc=True))),
    ("attention_fwd_simt_drop", "attention_fwd",
     lambda: ((*_attn(dtype=F32), 8, 2, 2, 4, 5), dict(use_tc=False, batch_major=True, drop=(-3, 51)))),
    ("attention_bwd_tc", "attention_bwd",
     lambda: ((*_attn(), t(16, 8, dtype=BF16), t(16, 24, dtype=BF16), t(16, 2), 8, 2, 2, 4, 5),
              dict(use_tc=True, drop=(2 ** 33 + 7, 26), dq_colsum=t(8), delta_token_major=True))),
    ("attention_bwd_simt", "attention_bwd",
     lambda: ((*_attn(dtype=F32), t(16, 8), t(16, 24), t(32), 8, 2, 2, 4, 0), dict(use_tc=False, batch_major=True))),
    ("attention_ctx_fwd_tc", "attention_ctx_fwd",
     lambda: ((t(8, 24, dtype=BF16), t(6, 16, dtype=BF16), t(8, 8, dtype=BF16), 4, 3, 2, 2, 4), dict(use_tc=True))),
    ("attention_ctx_fwd_simt", "attention_ctx_fwd",
     lambda: ((t(8, 24), t(6, 16), t(8, 8), 4, 3, 2, 2, 4), dict(use_tc=False))),
    ("attention_ctx_fwd_n0", "attention_ctx_fwd",
     lambda: ((t(8, 24, dtype=BF16), t(6, 16, dtype=BF16), t(8, 8, dtype=BF16), 4, 0, 2, 2, 4), dict(use_tc=True))),
    ("embed_fwd", "embed_fwd", lambda: ((t(6, 2, 3), t(6, 2), t(8, 3), t(8), t(8), t(8), t(12, 8, dtype=BF16),
                                         6, 2, 3, 8, 4), {})),
    ("embed_bwd_f1", "embed_bwd", lambda: ((t(12, 8), t(6, 2, 1), t(6, 2), t(8, 1), t(8), t(8), t(8), 6, 2, 1, 8, 4), {})),
    ("embed_bwd_f9", "embed_bwd", lambda: ((t(12, 8, dtype=BF16), t(6, 2, 9), t(6, 2), t(8, 9), t(8), t(8), t(8),
                                            6, 2, 9, 8, 4), {})),
    ("layernorm_fwd", "layernorm_fwd", lambda: ((t(5, 8, dtype=BF16), t(8), t(8), t(5, 8, dtype=BF16), t(5), t(5)),
                                                dict(eps=1e-6))),
    ("layernorm_bwd", "layernorm_bwd", lambda: ((t(5, 8), t(5, 8), t(5), t(5), t(8), t(5, 8), t(8), t(8)), {})),
    ("layernorm_bwd_colsum", "layernorm_bwd",
     lambda: ((t(5, 8, dtype=BF16), t(5, 8, dtype=BF16), t(5), t(5), t(8), t(5, 8, dtype=BF16), t(8), t(8)),
              dict(colsum_out=t(8)))),
    ("colsum", "colsum", lambda: ((t(7, 10, dtype=BF16), t(10)), {})),
    ("colsum_n", "colsum", lambda: ((t(7, 10), t(6)), dict(N=6))),
    ("bar_nll_fwd", "bar_nll_fwd", lambda: ((t(5, 12, dtype=BF16), t(5), t(11), 10, True, t(5), t(5, dtype=I64), t(5),
                                             t(1, dtype=I32)), {})),
    ("bar_nll_bwd", "bar_nll_bwd", lambda: ((t(5, 12), t(5, dtype=I64), t(5), t(5), t(5, 16, dtype=BF16), 10),
                                            dict(n_cols_pad=16))),
    ("bar_bucket_idx", "bar_bucket_idx", lambda: ((t(3, 4), t(11), 10, t(3, 4, dtype=I64)), {})),
    ("dropout_residual", "dropout", lambda: ((t(4, 6, dtype=BF16), t(4, 6, dtype=BF16), 2 ** 32 + 9, 51),
                                             dict(residual=t(4, 6, dtype=BF16)))),
    ("dropout", "dropout", lambda: ((t(4, 6), t(4, 6), -1, 0), {})),
    ("dropout_keep_mask", "dropout_keep_mask", lambda: ((t(4, 6, dtype=U8), 2 ** 40 + 11, 64), {})),
    ("adam_chunk_elems", "adam_chunk_elems", lambda: ((), {})),
    ("adam_step_clip", "adam_step", lambda: ((t(3, 6, dtype=I64), t(4, dtype=I32), 3, 4, 1e-3, 0.9, 0.999, 1e-8, 0.01,
                                              1.0, 7, t(1)), {})),
    ("adam_step", "adam_step", lambda: ((t(3, 6, dtype=I64), t(4, dtype=I32), 3, 4, 1e-3, 0.9, 0.999, 1e-8, 0.0, 0.0,
                                         1, t(1)), {})),
    ("gp_sample", "gp_sample", lambda: ((t(2, 5, 3), t(2, 5), t(2, 3), t(2), t(2), 1e-6, L.KERNEL_MATERN32, t(2, 5),
                                         t(2, 25), t(2, dtype=I32)), {})),
    ("gp_fit", "gp_fit", lambda: ((t(2, 6, 3), t(2, 6), L.gp_fit_desc(2, 6, 3, [3, 5], L.KERNEL_RBF, _gp_hyper(), 1e-4,
                                                                       1e-2, 50, 60, 1e-9, 1e-5),
                                   t(4, 6, dtype=F64), t(4, dtype=F64), t(4, dtype=I32), t(4, dtype=I32),
                                   t(4, dtype=I32)),
                                  dict(theta0=t(6, dtype=F64), grad=t(4, 6, dtype=F64), mean=t(4, dtype=F64),
                                       var=t(4, dtype=F64)))),
    ("gp_fit_bare", "gp_fit", lambda: ((t(2, 6, 3), t(2, 6), L.gp_fit_desc(2, 6, 3, [4], L.KERNEL_MATERN12, _gp_hyper(),
                                                                            1e-4, 1e-2, 50, 60, 1e-9, 1e-5),
                                        t(2, 6, dtype=F64), t(2, dtype=F64), t(2, dtype=I32), t(2, dtype=I32),
                                        t(2, dtype=I32)), {})),
    ("gp_mcmc", "gp_mcmc", lambda: ((t(2, 6, 3), t(2, 6), L.gp_mcmc_desc(2, 6, 3, [3, 5], L.KERNEL_MATERN52,
                                                                         _gp_hyper(), 4, 2, -5, n_pred=2),
                                     t(4, 4, 5, dtype=F64), t(4, dtype=F64), t(4, dtype=F64), t(4, 6, dtype=I32)),
                                    dict(init=t(4, 5, dtype=F64), log_samples=t(4, 4, 5, dtype=F64),
                                         mean=t(4, 4, 2, dtype=F64), var=t(4, 4, 2, dtype=F64), potential=t(4, dtype=F64),
                                         grad=t(4, 5, dtype=F64), trace=t(4, 6, 7, dtype=F64)))),
    ("gp_mcmc_bare", "gp_mcmc", lambda: ((t(1, 6, 3), t(1, 6), L.gp_mcmc_desc(1, 6, 3, [], L.KERNEL_RBF, _gp_hyper(),
                                                                              4, 2, 2 ** 32 + 1),
                                          t(1, 4, 5, dtype=F64), t(1, dtype=F64), t(1, dtype=F64),
                                          t(1, 6, dtype=I32)), {})),
    ("stroke_geometry", "stroke_geometry", lambda: ((_stroke_desc(), -2, t(2, 3, 4, 4, dtype=I32),
                                                     t(2, 3, 4, dtype=F64), t(1, dtype=I32)), {})),
    ("stroke_render", "stroke_render", lambda: ((_stroke_desc(), 2 ** 35, t(6, 2, dtype=I32), t(2, 3, 4, 4, dtype=I32),
                                                 t(2, 3, 4, dtype=F64), t(6, 2, 784), True), {})),
    ("stroke_raster", "stroke_raster", lambda: ((t(3, 4, 4, dtype=I32), t(3, dtype=I32), t(3, dtype=I32),
                                                 t(3, 400, dtype=U8), t(3, 400, dtype=U8), t(3, 400, dtype=U8), 20), {})),
    ("omniglot_episodes", "omniglot_episodes", lambda: ((_omniglot_desc(), 2 ** 33 + 3, t(10, 20, 28, 28, dtype=U8),
                                                         t(2, dtype=I32), t(6, 2, 784), t(6, 2, dtype=I64),
                                                         t(6, 2, dtype=I64)), {})),
    ("bnn_prior", "bnn_prior", lambda: ((t(5, 2, 3), t(5, 2), -7, 4), dict(dataset_offset=3, weights=t(2, 26),
                                                                          x_raw=t(5, 2, 3), u=t(5, 2, dtype=F64)))),
    ("bnn_prior_bare", "bnn_prior", lambda: ((t(5, 2, 3), t(5, 2), 9, 4), {})),
    ("bnn_mcmc_workspace", "bnn_mcmc_workspace", lambda: ((L.bnn_mcmc_desc(2, 5, 3, 2, 4, 6, 3, 2 ** 32 + 2),), {})),
    ("bnn_mcmc", "bnn_mcmc", lambda: ((t(2, 5, 2), t(2, 5), t(2, 3, 2), L.bnn_mcmc_desc(2, 5, 3, 2, 4, 6, 3, -9,
                                                                                         max_tree_depth=6),
                                       t(2, 6, 22, dtype=F64), t(2, dtype=F64), t(2, dtype=F64), t(2, 6, dtype=I32)),
                                      dict(init=t(2, 22, dtype=F64), probs=t(2, 6, 3, dtype=F64), obs=t(2, 6, 3),
                                           potential=t(2, dtype=F64), grad=t(2, 22, dtype=F64),
                                           trace=t(2, 9, 24, dtype=F64), workspace=t(2, 40, dtype=F64)))),
    ("bnn_mcmc_bare", "bnn_mcmc", lambda: ((t(2, 5, 2), t(2, 5), None, L.bnn_mcmc_desc(2, 5, 0, 2, 4, 6, 3, 1),
                                            t(2, 6, 22, dtype=F64), t(2, dtype=F64), t(2, dtype=F64),
                                            t(2, 6, dtype=I32)), {})),
    ("knn_cv", "knn_cv", lambda: ((t(9, 2, 3), t(6, 2), t(3, 2, dtype=F64), t(2, dtype=I32), t(2, 4, dtype=F64),
                                   t(2, dtype=I32)), {})),
    ("ridge_prefix", "ridge_prefix", lambda: ((t(2, 6, 3), t(2, 6), t(2, 6), 0.5, t(2, 6, dtype=F64),
                                               t(2, 6, dtype=F64)), {})),
    ("exact_gp_evaluate", "exact_gp_evaluate", lambda: ((t(2, 6, 3), t(2, 6), 0.6, 1e-4, t(2, 6, dtype=F64),
                                                         t(2, 6, dtype=F64), t(2, dtype=I32)), {})),
    ("exact_gp_sample", "exact_gp_sample", lambda: ((t(2, 6, 3), t(2, 6), 0.6, t(2, 6), t(2, dtype=I32)),
                                                    dict(factor=t(2, 6, 6, dtype=F64), perm=t(2, 6, dtype=I32)))),
    ("exact_gp_sample_bare", "exact_gp_sample", lambda: ((t(2, 6, 3), t(2, 6), 0.6, t(2, 6), t(2, dtype=I32)), {})),
    ("conv_fwd", "conv_fwd", lambda: ((t(2, 10, 10, 1), t(64, 1, 3, 3, dtype=BF16), t(64), t(2, 8, 8, 64, dtype=BF16),
                                       2, 10, 1), {})),
    ("conv_dgrad", "conv_dgrad", lambda: ((t(2, 12, 12, 64), t(64, 64, 3, 3), t(2, 8, 8, 64), t(2, 12, 12, 64), 2, 8),
                                          {})),
    ("conv_wgrad_workspace", "conv_wgrad_workspace", lambda: ((2, 10, 64), {})),
    ("conv_wgrad", "conv_wgrad", lambda: ((t(2, 12, 12, 64, dtype=BF16), t(2, 10, 10, 64, dtype=BF16),
                                           t(64, 64, 3, 3), t(64), 2, 10, 64), {})),
    ("conv_mean_fwd", "conv_mean_fwd", lambda: ((t(2, 4, 4, 64, dtype=BF16), t(2, 64), 2, 4), {})),
    ("conv_mean_bwd", "conv_mean_bwd", lambda: ((t(2, 64), t(2, 4, 4, 64), t(2, 8, 8, 64), 2, 4), {})),
    ("scaled_head_fwd", "scaled_head_fwd", lambda: ((t(5, 20), 9, t(5, 12), t(5)), {})),
    ("scaled_head_bwd", "scaled_head_bwd", lambda: ((t(5, 12), t(5, 20), t(5), 9, t(5, 24, dtype=BF16)),
                                                    dict(n_cols_pad=24))),
    ("scaled_head_bwd_default_pad", "scaled_head_bwd", lambda: ((t(5, 12), t(5, 20), t(5), 9, t(5, 20)), {})),
    ("fixed_scaled_head_fwd", "fixed_scaled_head_fwd", lambda: ((t(5, 12), 9, t(50), t(5, 12), t(1)), {})),
    ("fixed_scaled_head_bwd", "fixed_scaled_head_bwd", lambda: ((t(5, 12), t(5, 12), t(1), 9, t(5, 16, dtype=BF16),
                                                                 t(50)), dict(n_cols_pad=16, row_dot=t(5)))),
    ("fixed_scaled_head_bwd_scratch", "fixed_scaled_head_bwd", lambda: ((t(5, 12), t(5, 12), t(1), 9, t(5, 12), t(50)),
                                                                        {})),
    ("fixed_scaled_head_bwd_0rows", "fixed_scaled_head_bwd", lambda: ((t(0, 12), t(0, 12), t(1), 9, t(0, 16), t(50)),
                                                                      dict(n_cols_pad=16))),
]
CASE_IDS = [c[0] for c in CASES]


def _tensor_names(fn, args, kwargs):
    """{id(tensor): name} of the tensor arguments of one call (an element of a tuple argument as `name[i]`)."""
    names = {}
    for name, v in inspect.signature(fn).bind(*args, **kwargs).arguments.items():
        for i, x in (enumerate(v) if isinstance(v, tuple) else [(None, v)]):
            if torch.is_tensor(x):
                names.setdefault(id(x), name if i is None else f"{name}[{i}]")
    return names


def _spans(fn, args, kwargs):
    """(name, first byte, end byte) of every tensor argument, in argument order."""
    tensors = {id(x): x for v in list(args) + list(kwargs.values()) for x in (v if isinstance(v, tuple) else (v,))
               if torch.is_tensor(x)}
    spans = []
    for i, name in _tensor_names(fn, args, kwargs).items():
        s = tensors[i].untyped_storage()
        spans.append((name, tensors[i].data_ptr(), s.data_ptr() + s.nbytes()))
    return spans


def _pointer(p, spans):
    if isinstance(p, ctypes.c_void_p):
        p = p.value
    if not p:
        return None
    for name, lo, _ in spans:
        if p == lo:
            return f"{name}+0"
    for name, lo, hi in spans:
        if lo <= p < hi:
            return f"{name}+{p - lo}"
    return "<not an argument>"


def _struct(d, spans):
    out = {}
    for name, ctype in d._fields_:
        v = getattr(d, name)
        if ctype is ctypes.c_void_p:
            v = _pointer(v, spans)
        elif issubclass(ctype, ctypes._Pointer):
            v = [v[i] for i in range(getattr(d, "n_" + name))]
        out[name] = v
    return out


def _decode(a, spans):
    if a is STREAM:
        return "<stream>"
    if isinstance(a, ctypes.c_void_p):
        return _pointer(a, spans)
    if type(a).__name__ == "CArgObject":                # ctypes.byref(descriptor)
        return {"byref": _struct(a._obj, spans)}
    if a is None or isinstance(a, (bool, int, float)):
        return a
    raise TypeError(f"cannot decode {type(a)}")


class FakeLib:
    """One recording function per `_PROTOTYPES` entry: launches return 0, the queries a fixed positive count."""

    def __init__(self):
        self.calls, self.spans = [], []
        for name in L._PROTOTYPES:
            setattr(self, name, self._entry(name))

    def _entry(self, name):
        def f(*args):
            self.calls.append({"fn": name, "args": [_decode(a, self.spans) for a in args]})
            return b"fake" if name == "pfn_last_error" else QUERIES.get(name, 0)
        return f


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(L, "load", lambda: lib)
    monkeypatch.setattr(L, "stream_ptr", lambda device=None: STREAM)
    return lib


def _record(case, lib, monkeypatch):
    """The log entry of one case: entry points and decoded arguments, launches counted, tensors checked."""
    _, wrapper, build = next(c for c in CASES if c[0] == case)
    fn = getattr(L, wrapper)
    args, kwargs = build()
    names = _tensor_names(fn, args, kwargs)
    checked = set()
    monkeypatch.setattr(L, "require_cuda",
                        lambda *ts: checked.update(names[id(x)] for x in ts if x is not None and id(x) in names))
    lib.calls, lib.spans = [], _spans(fn, args, kwargs)
    n0 = L.launch_count()
    fn(*args, **kwargs)
    return {"calls": lib.calls, "launches": L.launch_count() - n0, "require_cuda": sorted(checked)}


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("case", CASE_IDS)
def test_call_log_matches_golden(case, fake, monkeypatch):
    assert _record(case, fake, monkeypatch) == _golden()[case]


def test_cases_cover_every_wrapper_and_entry_point():
    golden = _golden()
    assert list(golden) == CASE_IDS
    called = {c["fn"] for entry in golden.values() for c in entry["calls"]}
    assert called == set(L._PROTOTYPES) - NOT_CALLED
    guarded = {name for name, f in vars(L).items()
               if isinstance(f, types.FunctionType) and hasattr(f, "__wrapped__") and not name.startswith("_")}
    queries = {"adam_chunk_elems", "bnn_mcmc_workspace", "conv_wgrad_workspace"}
    assert guarded | queries <= {c[1] for c in CASES}


def _fake_cuda(args, kwargs):
    """`args` and `kwargs` with every tensor replaced by an unbacked one of the same shape, stride and dtype on cuda:0."""
    from torch._subclasses.fake_tensor import FakeTensorMode
    with FakeTensorMode():
        def conv(x):
            if isinstance(x, tuple):
                return tuple(conv(y) for y in x)
            if torch.is_tensor(x):
                return torch.empty_strided(x.shape, x.stride(), dtype=x.dtype, device="cuda")
            return x
        return [conv(a) for a in args], {k: conv(v) for k, v in kwargs.items()}


@pytest.mark.parametrize("case", CASE_IDS)
def test_cpu_tensor_is_rejected_before_the_library_is_called(case, fake):
    """Each tensor argument in turn on the CPU, the others on a CUDA device: the call raises require_cuda's error, the
    library is not called and no launch is counted.  attention_ctx_fwd's kv with n == 0 is not read and not checked."""
    _, wrapper, build = next(c for c in CASES if c[0] == case)
    fn = getattr(L, wrapper)
    args, kwargs = build()
    cuda_args, cuda_kwargs = _fake_cuda(args, kwargs)
    probes = [(i, None) for i, a in enumerate(args) if torch.is_tensor(a)]
    probes += [(k, None) for k, v in kwargs.items() if torch.is_tensor(v)]
    probes += [(k, j) for k, v in kwargs.items() if isinstance(v, tuple) for j, x in enumerate(v) if torch.is_tensor(x)]
    if case == "attention_ctx_fwd_n0":
        probes.remove((1, None))
    for key, j in probes:
        a, kw = list(cuda_args), dict(cuda_kwargs)
        where = a if isinstance(key, int) else kw
        src = args if isinstance(key, int) else kwargs
        if j is None:
            where[key] = src[key]
        else:
            where[key] = tuple(src[key][m] if m == j else x for m, x in enumerate(where[key]))
        fake.calls = []
        n0 = L.launch_count()
        with pytest.raises(RuntimeError, match="sm_90a CUDA kernels only"):
            fn(*a, **kw)
        assert fake.calls == [] and L.launch_count() == n0, (case, key, j)


def write_golden():
    mp = pytest.MonkeyPatch()
    try:
        lib = FakeLib()
        mp.setattr(L, "load", lambda: lib)
        mp.setattr(L, "stream_ptr", lambda device=None: STREAM)
        log = {case: _record(case, lib, mp) for case in CASE_IDS}
    finally:
        mp.undo()
    with open(GOLDEN, "w") as f:
        json.dump(log, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    write_golden()
