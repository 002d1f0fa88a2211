"""The engine's three decoder heads (DecoderFn, ScaledDecoderFn, FixedScaledDecoderFn) forward and backward on the CPU,
through an fp64 recording fake of the kernel library: the literal call plan of each head (function, GEMM epilogue,
accumulate, split-K, output shape, row pitch and dtype), the one gradient bucket each head reports and its layout, and
the logits and gradients against the fp64 restatements (oracle/decoders_oracle.py, and autograd for the default head)."""
import pytest
import torch

from oracle import decoders_oracle as DO
from transformerscandobayesianinference_b200 import _lib, engine

NQ, E, NHID, NOUT, NT = 37, 16, 24, 9, 50          # NOUT pads to 12 (fp32 rows) and to 16 (activation-dtype rows)
NZ = NOUT + _lib.HEAD_TEMPS                        # 19: pads to 20 and to 24
F32 = torch.float32
DTYPES = {"bf16": torch.bfloat16, "fp32": F32}
EPI_NAMES = {_lib.EPI_NONE: "none", _lib.EPI_GELU: "gelu", _lib.EPI_GELU_BWD: "gelu_bwd", _lib.EPI_MUL: "mul"}


def _out(t):
    """What the plan records of a written buffer: shape, row pitch (2-D) and dtype."""
    return tuple(t.shape), t.stride(0) if t.dim() == 2 else None, t.dtype


class FakeLib:
    """The library entry points the heads call, restated in fp64 and stored in each output's dtype; every call is
    appended to `calls`, and so are the data-parallel hook and sync."""
    EPI_NONE, EPI_GELU, EPI_GELU_BWD, EPI_MUL = _lib.EPI_NONE, _lib.EPI_GELU, _lib.EPI_GELU_BWD, _lib.EPI_MUL
    HEAD_TEMPS = _lib.HEAD_TEMPS

    def __init__(self):
        self.calls = []

    def require_cuda(self, *tensors):
        pass

    def num_sms(self, device=None):
        return 132

    def tc_gemm_ok(self, A, B, *rest):
        return A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16

    def gemm(self, A, B, C, *, a_mn_major=False, b_mn_major=False, bias=None, aux=None, C2=None, epilogue=EPI_NONE,
             accumulate=False, k_splits=1, M=None, N=None, K=None, use_tc=None, rowdot=None, c2_gelu_grad=False):
        sig = "gemm/" + EPI_NAMES[epilogue] + ("/acc" if accumulate else "")
        self.calls.append((sig, k_splits, _out(C)))
        y = (A.t() if a_mn_major else A).double() @ (B.t() if b_mn_major else B).double().t()
        if bias is not None:
            y = y + bias.double()
        if epilogue == self.EPI_GELU:
            C2.copy_(DO.gelu_grad(y) if c2_gelu_grad else y)
            y = DO.gelu(y)
        elif epilogue == self.EPI_GELU_BWD:
            y = y * DO.gelu_grad(aux.double())
        elif epilogue == self.EPI_MUL:
            y = y * aux.double()
        elif aux is not None:
            y = y + aux.double()
        C.copy_(C.double() + y if accumulate else y)

    def colsum(self, X, out, N=None):
        self.calls.append(("colsum", _out(out)))
        out += X.double().sum(0).to(out.dtype)

    def scaled_head_fwd(self, zz, n_out, out, temp):
        self.calls.append(("scaled_head_fwd", _out(out), _out(temp)))
        o, t, _ = DO.scaled_rows(zz, n_out)
        out.copy_(o)
        temp.copy_(t)

    def scaled_head_bwd(self, g, zz, temp, n_out, dzz, n_cols_pad=None):
        self.calls.append(("scaled_head_bwd", _out(dzz)))
        nz = n_out + self.HEAD_TEMPS
        dzz[:, :nz] = DO.scaled_rows_bwd(g, zz, n_out).to(dzz.dtype)
        dzz[:, nz:n_cols_pad] = 0

    def fixed_scaled_head_fwd(self, z, n_out, T, out, S):
        self.calls.append(("fixed_scaled_head_fwd", _out(out), _out(S)))
        S.fill_(T.double().sum().item())
        out.copy_(z.double() / S.double())

    def fixed_scaled_head_bwd(self, g, z, S, n_out, dz, dT, n_cols_pad=None, row_dot=None):
        self.calls.append(("fixed_scaled_head_bwd", _out(dz), _out(dT)))
        s = S.double().item()
        dz[:, :n_out] = (g.double() / s).to(dz.dtype)
        dz[:, n_out:n_cols_pad] = 0
        dT.fill_(-(g.double() * z.double()).sum().item() / s ** 2)


def _run(fn, inputs, precision, n_outputs=1):
    """fn.apply forward and backward (gradient seeded from NQ) on the fake: (forward calls, backward calls, outputs,
    the output gradient, the input gradients, the buckets reported)."""
    lib = FakeLib()
    buckets = []
    hq = torch.randn(NQ, E, generator=torch.Generator().manual_seed(NQ)).to(DTYPES[precision]).requires_grad_()
    params = [p.detach().clone().requires_grad_() for p in inputs]
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(engine, "L", lib)
        mp.setattr(engine, "_GELU_GRAD_FWD", True)
        mp.setattr(engine, "GRAD_BUCKET_HOOK", lambda flat: (lib.calls.append("hook"), buckets.append(flat.clone())))
        mp.setattr(engine, "GRAD_BUCKET_SYNC", lambda: lib.calls.append("sync"))
        out = fn.apply(hq, *params, precision)
        n_fwd = len(lib.calls)
        logits = out[0] if n_outputs > 1 else out
        gout = torch.randn(logits.shape, generator=torch.Generator().manual_seed(7), dtype=torch.float64)
        logits.backward(gout.float())
    return (lib.calls[:n_fwd], lib.calls[n_fwd:], out, gout, hq.grad, [p.grad for p in params], hq.detach(), buckets)


def _mlp_plan(precision, first_out):
    """The shared part of each head's backward: the second layer's bias and weight gradients, the GELU layer's dgrad,
    its bias and weight gradients, the input gradient; `first_out` rows of the second layer."""
    dt = DTYPES[precision]
    return [("colsum", ((first_out,), None, F32)), ("gemm/none/acc", 1, ((first_out, NHID), NHID, F32)),
            ("gemm/mul" if precision == "bf16" else "gemm/gelu_bwd", 1, ((NQ, NHID), NHID, dt)),
            ("colsum", ((NHID,), None, F32)), ("gemm/none/acc", 1, ((NHID, E), E, F32)),
            ("gemm/none", 1, ((NQ, E), E, dt)), "hook", "sync"]


def _gelu_call(precision):
    return ("gemm/gelu", 1, ((NQ, NHID), NHID, DTYPES[precision]))


def _weights(seed, *shapes):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=g) * (s[-1] ** -0.5 if len(s) == 2 else 0.1) for s in shapes]


def _close(got, want, precision, what):
    rtol = 3e-2 if precision == "bf16" else 1e-4
    err = (got.double() - want.double()).abs().max().item()
    assert err <= rtol * want.double().abs().max().item() + 1e-12, f"{what}: max error {err}"


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_default_head(precision):
    W0, b0, W2, b2 = _weights(1, (NHID, E), (NHID,), (NOUT, NHID), (NOUT,))
    fwd, bwd, logits, gout, dhq, grads, hq, buckets = _run(engine.DecoderFn, (W0, b0, W2, b2), precision)
    assert fwd == [_gelu_call(precision), ("gemm/none", 1, ((NQ, NOUT), 12, F32))]
    assert bwd == _mlp_plan(precision, NOUT)
    assert len(buckets) == 1 and torch.equal(buckets[0], torch.cat([g.flatten() for g in grads]))
    x = hq.double().requires_grad_()
    ref = [t.double().requires_grad_() for t in (W0, b0, W2, b2)]
    want = torch.nn.functional.gelu(x @ ref[0].T + ref[1]) @ ref[2].T + ref[3]
    want.backward(gout)
    _close(logits, want.detach(), precision, "logits")
    _close(dhq, x.grad, precision, "dhq")
    for name, g, r in zip(("dW0", "db0", "dW2", "db2"), grads, ref):
        _close(g, r.grad, precision, name)


def test_default_head_keeps_autograds_in_place_check():
    """DecoderFn saves W0 and W2 with save_for_backward: an in-place edit between forward and backward raises."""
    W0, b0, W2, b2 = (p.requires_grad_() for p in _weights(1, (NHID, E), (NHID,), (NOUT, NHID), (NOUT,)))
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(engine, "L", FakeLib())
        logits = engine.DecoderFn.apply(torch.randn(NQ, E), W0, b0, W2, b2, "fp32")
        with torch.no_grad():
            W2.mul_(2)
        with pytest.raises(RuntimeError, match="modified by an inplace operation"):
            logits.sum().backward()


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_scaled_head(precision):
    W, b, W1, b1, W2, b2 = _weights(2, (NHID, E), (NHID,), (NOUT, NHID), (NOUT,), (DO.N_TEMPS, NHID), (DO.N_TEMPS,))
    W2 = W2 * 8                                                  # spread the temperature softmax
    fwd, bwd, (logits, temp), gout, dhq, grads, hq, buckets = _run(engine.ScaledDecoderFn, (W, b, W1, b1, W2, b2),
                                                                   precision, 2)
    assert fwd == [_gelu_call(precision), ("gemm/none", 1, ((NQ, NZ), 20, F32)),
                   ("scaled_head_fwd", ((NQ, NOUT), 12, F32), ((NQ,), None, F32))]
    assert bwd == [("scaled_head_bwd", ((NQ, 24), 24, DTYPES[precision]))] + _mlp_plan(precision, NZ)
    # the bucket holds the stacked second layer: [W1; W2] then [b1; b2]
    dW, db, dW1, db1, dW2, db2 = grads
    assert len(buckets) == 1 and torch.equal(buckets[0], torch.cat([t.flatten() for t in (dW, db, dW1, dW2, db1, db2)]))
    r = DO.scaled_head(hq, W, b, W1, b1, W2, b2, gout)
    _close(logits, r["out"], precision, "logits")
    _close(temp, r["temp"], precision, "temp")
    _close(dhq, r["dhq"], precision, "dhq")
    names = ("linear.weight", "linear.bias", "linear1.weight", "linear1.bias", "linear2.weight", "linear2.bias")
    for name, g in zip(names, grads):
        _close(g, r["grads"][name], precision, name)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_fixed_scaled_head(precision):
    W0, b0, W2, b2 = _weights(3, (NHID, E), (NHID,), (NOUT, NHID), (NOUT,))
    T = torch.rand(NT, generator=torch.Generator().manual_seed(4)) * 0.1
    fwd, bwd, logits, gout, dhq, grads, hq, buckets = _run(engine.FixedScaledDecoderFn, (W0, b0, W2, b2, T), precision)
    assert fwd == [_gelu_call(precision), ("gemm/none", 1, ((NQ, NOUT), 12, F32)),
                   ("fixed_scaled_head_fwd", ((NQ, NOUT), 12, F32), ((1,), None, F32))]
    assert bwd == [("fixed_scaled_head_bwd", ((NQ, 16), 16, DTYPES[precision]), ((NT,), None, F32))] \
        + _mlp_plan(precision, NOUT)
    assert len(buckets) == 1 and torch.equal(buckets[0], torch.cat([g.flatten() for g in grads]))
    r = DO.fixed_head(hq, W0, b0, W2, b2, T, gout)
    _close(logits, r["out"], precision, "logits")
    _close(dhq, r["dhq"], precision, "dhq")
    for name, g in zip(("mapper.0.weight", "mapper.0.bias", "mapper.2.weight", "mapper.2.bias", "T"), grads):
        _close(g, r["grads"][name], precision, name)
