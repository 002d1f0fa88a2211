"""encoders.Conv on the host: its parameters, shapes and argument checks, the fp64 oracle against torch's own Conv2d
module, and each kernel bound of oracle/conv_oracle.py against the exact result and seeded slips."""
import pytest
import torch
import torch.nn as nn

from oracle import conv_oracle as co
from oracle import error_budget as eb
from transformerscandobayesianinference_b200 import encoders


def test_parameters_and_state_dict_keys():
    m = encoders.Conv(784, 512)
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    expect = {}
    for i in range(5):
        expect[f"convs.{i}.weight"] = (64, 1 if i == 0 else 64, 3, 3)
        expect[f"convs.{i}.bias"] = (64,)
    expect["linear.weight"], expect["linear.bias"] = (512, 64), (512,)
    assert shapes == expect and list(shapes) == list(expect)


def test_seeded_construction_equals_the_torch_module():
    torch.manual_seed(3)
    m = encoders.Conv(784, 32)
    torch.manual_seed(3)
    convs = nn.ModuleList([nn.Conv2d(1 if i == 0 else 64, 64, 3) for i in range(5)])
    linear = nn.Linear(64, 32)
    ref = dict(convs=convs, linear=linear)
    for k, v in m.state_dict().items():
        head, rest = k.split(".", 1)
        assert torch.equal(v, ref[head].state_dict()[rest]), k


@pytest.mark.parametrize("S,n", [(4, 1), (5, 1), (6, 2), (7, 2), (12, 5), (28, 5), (105, 5), (112, 5)])
def test_n_conv(S, n):
    assert encoders.Conv(S * S, 8).n_conv == n == co.n_conv(S)


@pytest.mark.parametrize("size", [783, 3 * 3, 113 * 113, 10, 0])
def test_rejects_bad_sizes(size):
    with pytest.raises(ValueError):
        encoders.Conv(size, 8)


def test_rejects_input_gradient_and_cpu_tensors():
    m = encoders.Conv(36, 8)
    with pytest.raises(ValueError):
        m(torch.rand(2, 36, requires_grad=True))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.rand(2, 36))


@pytest.mark.parametrize("S", [4, 6, 9, 13])
def test_oracle_matches_torch_module_in_fp64(S):
    torch.manual_seed(S)
    m = encoders.Conv(S * S, 16).double()
    x = torch.rand(5, S * S, dtype=torch.float64)
    h = x.reshape(-1, 1, S, S)
    for c in m.convs[:m.n_conv]:
        h = torch.relu(c(h))
    ref = m.linear(h.mean((2, 3)))
    params = [p for c in m.convs[:m.n_conv] for p in (c.weight, c.bias)] + [m.linear.weight, m.linear.bias]
    out, _, _ = co.forward(x, params, S)
    assert torch.allclose(out, ref, rtol=1e-12, atol=1e-14)
    dout = torch.randn(5, 16, dtype=torch.float64)
    ref.backward(dout)
    _, grads = co.gradients(x, params, S, dout)
    for p, g in zip(params, grads):
        assert torch.allclose(g, p.grad, rtol=1e-10, atol=1e-14)


# ---- the bounds against seeded slips ---------------------------------------------------------------------------------
def _bf16(t):
    return t.to(torch.bfloat16).double()


def _fails(name, got, exact, bound, c):
    with pytest.raises(AssertionError):
        eb.check(name, got, exact, bound, c, verbose=False)


def _layer(N=3, s=9, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = _bf16(torch.relu(torch.randn(N, s, s, 64, generator=g)))
    W = _bf16(torch.randn(64, 64, 3, 3, generator=g) / 24)
    b = torch.randn(64, generator=g).float() / 4
    return x, W, b, g


def test_fwd_bound_passes_exact_and_catches_slips():
    x, W, b, _ = _layer()
    exact, bound = co.conv_fwd(x, W, b, eb.U)
    eb.check("exact", _bf16(exact), exact, bound, co.C_CONV, verbose=False)
    Ws = W.clone()
    Ws[:, :, 1, 1], Ws[:, :, 1, 2] = W[:, :, 1, 2], W[:, :, 1, 1]      # centre tap read one pixel to the right
    _fails("tap shifted", _bf16(co.conv_fwd(x, Ws, b, eb.U)[0]), exact, bound, co.C_CONV)
    _fails("bias dropped", _bf16(co.conv_fwd(x, W, torch.zeros_like(b), eb.U)[0]), exact, bound, co.C_CONV)
    missing = _bf16(exact).clone()
    missing[-1, -1] = 0                                                  # last output row of the last tile not written
    _fails("last row missing", missing, exact, bound, co.C_CONV)


def test_dgrad_bound_passes_exact_and_catches_slips():
    x, W, _, g = _layer()
    s = x.shape[1]
    gpad = torch.zeros(3, s + 2, s + 2, 64, dtype=torch.float64)
    gpad[:, 2:s, 2:s] = _bf16(torch.randn(3, s - 2, s - 2, 64, generator=g))
    exact, bound = co.conv_dgrad(gpad, W, x, eb.U)
    eb.check("exact", _bf16(exact), exact, bound, co.C_CONV, verbose=False)
    other = _bf16(torch.relu(torch.randn(x.shape, generator=g)))        # the ReLU mask of another layer
    _fails("wrong mask", _bf16(co.conv_dgrad(gpad, W, other, eb.U)[0]), exact, bound, co.C_CONV)
    _fails("unflipped weights", _bf16(co.conv_dgrad(gpad, W.flip(2, 3), x, eb.U)[0]), exact, bound, co.C_CONV)


def test_wgrad_bound_passes_exact_and_catches_slips():
    x, _, _, g = _layer(N=4, s=12)
    s = x.shape[1]
    gr = _bf16(torch.randn(4, s - 2, s - 2, 64, generator=g))
    dw, db, bw, bb = co.conv_wgrad(gr, x)
    eb.check("exact dW", dw.float(), dw, bw, 1.0, verbose=False)
    eb.check("exact db", db.float(), db, bb, 1.0, verbose=False)
    _fails("bf16 accumulator", _bf16(dw), dw, bw, 1.0)
    xs = torch.roll(x, 1, dims=2)                                      # every tap one pixel off
    _fails("tap shifted", co.conv_wgrad(gr, xs)[0], dw, bw, 1.0)
    gm = gr.clone()
    gm[-1, -1] = 0                                                      # last output row left out of the sum
    _fails("last row missing", co.conv_wgrad(gm, x)[1], db, bb, 1.0)


def test_mean_bounds_pass_exact_and_catch_slips():
    x, _, _, g = _layer(N=2, s=7)
    exact, bound = co.mean_fwd(x, eb.U)
    eb.check("exact", _bf16(exact), exact, bound, co.C_MEAN, verbose=False)
    _fails("last row missing", _bf16(x[:, :-1].reshape(2, -1, 64).sum(1) / 49), exact, bound, co.C_MEAN)
    dfeat = _bf16(torch.randn(2, 64, generator=g))
    gexact, gbound = co.mean_bwd(dfeat, x, eb.U)
    eb.check("exact", _bf16(gexact), gexact, gbound, co.C_MEAN, verbose=False)
    _fails("no mask", _bf16((dfeat / 49)[:, None, None, :].expand(x.shape)), gexact, gbound, co.C_MEAN)
