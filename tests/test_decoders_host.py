"""The learned-temperature decoder heads on the host: the fp64 restatement (oracle/decoders_oracle.py) against the
unmodified reference decoders.py, the modules' parameters and RNG behaviour, the drop-in registration, and the row
kernels' error bounds against float32 restatements of the kernels and seeded slips."""
import random
import sys

import pytest
import torch

from oracle import decoders_oracle as DO, error_budget as EB
from transformerscandobayesianinference_b200 import decoders, engine

F32 = torch.float32


@pytest.fixture(scope="module")
def ref():
    mod = DO.load_reference()
    if mod is None:
        pytest.skip("oracle/_ref has not been built (python oracle/build_ref.py)")
    return mod


def _head_input(rows, ninp, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(rows, ninp, generator=g, dtype=torch.float64)


# ------------------------------------------------------------------------------------------------------------------
# reference parity in float64 on the CPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nout", [1, 5, 100])
def test_scaled_restatement_matches_reference(ref, nout, monkeypatch):
    """The reference forms its temperatures with torch.tensor in the default dtype: run it with float64 as the default,
    so that its constants are the exact decimals, and give the restatement the same constants."""
    monkeypatch.setattr(random, "random", lambda: 0.0)
    torch.manual_seed(nout)
    m = ref.ScaledDecoder(16, 24, nout).double()
    with torch.no_grad():
        m.linear2.weight.mul_(8)                  # spread the temperature softmax
    x = _head_input(37, 16, 1).requires_grad_()
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        out = m(x)
    finally:
        torch.set_default_dtype(prev)
    gout = torch.randn_like(out)
    out.backward(gout)
    r = DO.scaled_head(x.detach(), m.linear.weight, m.linear.bias, m.linear1.weight, m.linear1.bias, m.linear2.weight,
                       m.linear2.bias, gout, temps=torch.tensor(DO.TEMPERATURES, dtype=torch.float64))
    torch.testing.assert_close(r["out"], out.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(r["dhq"], x.grad, rtol=1e-10, atol=1e-12)
    for name, p in m.named_parameters():
        torch.testing.assert_close(r["grads"][name], p.grad, rtol=1e-10, atol=1e-12, msg=name)


def test_fixed_restatement_matches_reference(ref):
    torch.manual_seed(3)
    m = ref.FixedScaledDecoder(16, 24, 7).double()
    with torch.no_grad():
        m.T.uniform_(0, 3e-4)
    x = _head_input(29, 16, 2).requires_grad_()
    out = m(x)
    gout = torch.randn_like(out)
    out.backward(gout)
    r = DO.fixed_head(x.detach(), *[p for _, p in m.named_parameters() if _ != "T"], m.T, gout)
    torch.testing.assert_close(r["out"], out.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(r["dhq"], x.grad, rtol=1e-10, atol=1e-12)
    for name, p in m.named_parameters():
        torch.testing.assert_close(r["grads"][name], p.grad, rtol=1e-10, atol=1e-12, msg=name)


# ------------------------------------------------------------------------------------------------------------------
# parameters, initialisation and the global random stream
# ------------------------------------------------------------------------------------------------------------------
def test_state_dict_keys_and_seeded_values_match_reference(ref):
    for cls in ("ScaledDecoder", "FixedScaledDecoder"):
        torch.manual_seed(11)
        ours = getattr(decoders, cls)(12, 20, 30).state_dict()
        torch.manual_seed(11)
        theirs = getattr(ref, cls)(12, 20, 30).state_dict()
        assert list(ours) == list(theirs), cls
        for k in ours:
            assert torch.equal(ours[k], theirs[k]), (cls, k)
        getattr(decoders, cls)(12, 20, 30).load_state_dict(theirs, strict=True)
        getattr(ref, cls)(12, 20, 30).load_state_dict(ours, strict=True)


def test_parameter_names():
    s = decoders.ScaledDecoder(4, 6, 3).state_dict()
    assert {k: tuple(v.shape) for k, v in s.items()} == {
        "linear.weight": (6, 4), "linear.bias": (6,), "linear1.weight": (3, 6), "linear1.bias": (3,),
        "linear2.weight": (10, 6), "linear2.bias": (10,)}
    f = decoders.FixedScaledDecoder(4, 6, 3).state_dict()
    assert list(f) == ["T", "mapper.0.weight", "mapper.0.bias", "mapper.2.weight", "mapper.2.bias"]
    assert f["T"].shape == (10000,) and torch.equal(f["T"], torch.ones(10000) / 10000)


def test_cpu_input_raises():
    for cls in (decoders.ScaledDecoder, decoders.FixedScaledDecoder):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            cls(4, 6, 3)(torch.randn(5, 4))


class _FakeFn:
    """Stands in for engine.ScaledDecoderFn on the host: logits of zeros, temp 1, 2, 3, ..."""
    @staticmethod
    def apply(h, W, b, W1, b1, W2, b2, precision):
        n = h.shape[0]
        return torch.zeros(n, W1.shape[0]), torch.arange(1, n + 1, dtype=F32)


@pytest.mark.parametrize("lead", [(6,), (3, 2), (2, 3, 2)])
def test_one_random_draw_per_forward_and_print_above_099(monkeypatch, capsys, lead):
    monkeypatch.setattr(engine, "ScaledDecoderFn", _FakeFn)
    m = decoders.ScaledDecoder(4, 6, 3)
    h = torch.zeros(int(torch.tensor(lead).prod()), 4)
    random.seed(5)
    want = [random.random() for _ in range(3)]
    random.seed(5)
    out = m.fused(h, lead, "fp32")
    assert out.shape == lead + (3,)
    assert random.random() == want[1]                 # exactly one draw was consumed
    assert capsys.readouterr().out == ""
    monkeypatch.setattr(random, "random", lambda: 0.995)
    m.fused(h, lead, "fp32")
    printed = capsys.readouterr().out
    temps = torch.arange(1, h.shape[0] + 1, dtype=F32).view(lead)
    assert printed.startswith(str(temps.shape)) and str((temps[:, :2] if len(lead) >= 2 else temps[:2])) in printed


def test_dropin_registers_decoders_and_model_builds():
    import transformerscandobayesianinference_b200 as pfn
    saved = {k: sys.modules.get(k) for k in ("decoders",) + pfn._DROPIN_MODULES}
    try:
        ret = pfn.install_dropin()
        assert set(ret) == set(pfn._DROPIN_MODULES)
        import decoders as d
        assert d is decoders
        from transformerscandobayesianinference_b200 import encoders, transformer
        m = transformer.TransformerModel(encoders.Linear(1, 32), 7, 32, 2, 48, 1, decoder=d.ScaledDecoder)
        names = [k for k in m.state_dict() if k.startswith("decoder.")]
        assert names == ["decoder.linear.weight", "decoder.linear.bias", "decoder.linear1.weight", "decoder.linear1.bias",
                         "decoder.linear2.weight", "decoder.linear2.bias"]
        assert m.decoder.linear1.out_features == 7 and m.decoder.linear.out_features == 48
        f = transformer.TransformerModel(encoders.Linear(1, 32), 7, 32, 2, 48, 1, decoder=d.FixedScaledDecoder)
        assert "decoder.T" in f.state_dict() and "decoder.mapper.2.weight" in f.state_dict()
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


# ------------------------------------------------------------------------------------------------------------------
# row-kernel bounds: float32 restatements of csrc/scaled_head.cu inside at c = 1, seeded slips outside at C_HEAD
# ------------------------------------------------------------------------------------------------------------------
def _butterfly(x):
    for o in (16, 8, 4, 2, 1):
        x = x + x[..., torch.arange(32) ^ o]
    return x[..., 0]


def _lanes(t, n):
    """[rows, n] -> [rows, ceil(n/32), 32] zero padded (lane i holds columns i, i + 32, ...)."""
    rows = t.shape[0]
    return torch.cat([t, torch.zeros(rows, (-n) % 32, dtype=t.dtype)], 1).view(rows, -1, 32)


def _fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def k_scaled_fwd(zz, n_out, temps=None):
    c = (DO.TEMPS if temps is None else temps).float()
    zt = zz[:, n_out:n_out + 10]
    e = torch.exp(zt - zt.max(-1, keepdim=True).values)
    p = e / _butterfly(torch.cat([e, torch.zeros(e.shape[0], 22)], 1)).unsqueeze(-1)
    t = _butterfly(torch.cat([p * c, torch.zeros(p.shape[0], 22)], 1))
    return zz[:, :n_out] / t.unsqueeze(-1), t, p


def k_scaled_bwd(g, zz, n_out, dtype, drop_factor=False):
    _, t, p = k_scaled_fwd(zz, n_out)
    gl, zl = _lanes(g, n_out), _lanes(zz[:, :n_out].contiguous(), n_out)
    s = torch.zeros(g.shape[0], 32)
    for j in range(gl.shape[1]):
        s = _fma(gl[:, j], zl[:, j], s)
    dtemp = -_butterfly(s) / (t * t)
    dz = g / t.unsqueeze(-1)
    fac = 1.0 if drop_factor else p * (DO.TEMPS.float() - t.unsqueeze(-1))
    return torch.cat([dz, fac * dtemp.unsqueeze(-1)], -1).to(dtype)


def k_fixed(g, z, T, dtype):
    """fp32 sums in torch's order, whose depth is below the kernels'."""
    S = T.sum()
    D = (g * z).sum()
    return z / S, S, (g / S).to(dtype), -D / (S * S)


def _zz(rows, n_out, seed, spread=3.0):
    gen = torch.Generator().manual_seed(seed)
    zz = torch.randn(rows, n_out + 10, generator=gen)
    zz[:, n_out:] *= spread
    return zz, torch.randn(rows, n_out, generator=gen)


def _ratio(got, exact, bound):
    err = (got.double() - exact.double()).abs()
    return (err / bound.double().clamp_min(1e-300)).masked_fill(bound == 0, 0.0).max().item()


@pytest.mark.parametrize("n_out,dtype", [(1, F32), (5, torch.bfloat16), (100, F32), (1000, torch.bfloat16)])
def test_scaled_restatement_inside_bound_at_c1(n_out, dtype):
    zz, g = _zz(33, n_out, n_out)
    u_d = EB.U32 if dtype == F32 else EB.U
    out, t, _ = k_scaled_fwd(zz, n_out)
    f = DO.scaled_fwd_bound(zz, n_out)
    EB.check("host scaled out", out, f["out"], f["out_bound"], 1.0)
    EB.check("host scaled temp", t, f["temp"], f["temp_bound"], 1.0)
    exact, bound = DO.scaled_bwd_bound(g, zz, n_out, u_d)
    EB.check("host scaled dzz", k_scaled_bwd(g, zz, n_out, dtype), exact, bound, 1.0)


def test_fixed_restatement_inside_bound_at_c1():
    zz, g = _zz(40, 30, 7)
    T = torch.rand(10240, generator=torch.Generator().manual_seed(1)) * 2e-4
    out, S, dz, dT = k_fixed(g, zz[:, :30], T, torch.bfloat16)
    f = DO.fixed_fwd_bound(zz[:, :30], T)
    EB.check("host fixed out", out, f["out"], f["out_bound"], 1.0)
    EB.check("host fixed S", S, f["S"], f["S_bound"], 1.0)
    b = DO.fixed_bwd_bound(g, zz[:, :30], S, EB.U)
    EB.check("host fixed dz", dz, b["dz"], b["dz_bound"], 1.0)
    EB.check("host fixed dT", dT, b["dT"], b["dT_bound"], 1.0)


def test_slip_wrong_temperature_constant():
    zz, _ = _zz(64, 20, 3)
    wrong = DO.TEMPS.clone()
    wrong[1] = 1.5
    out, t, _ = k_scaled_fwd(zz, 20, wrong)
    f = DO.scaled_fwd_bound(zz, 20)
    assert _ratio(t, f["temp"], f["temp_bound"]) > DO.C_HEAD
    assert _ratio(out, f["out"], f["out_bound"]) > DO.C_HEAD


@pytest.mark.parametrize("dtype", [F32, torch.bfloat16])
def test_slip_missing_softmax_factor(dtype):
    zz, g = _zz(64, 20, 4)
    exact, bound = DO.scaled_bwd_bound(g, zz, 20, EB.U32 if dtype == F32 else EB.U)
    got = k_scaled_bwd(g, zz, 20, dtype, drop_factor=True)
    assert _ratio(got[:, 20:], exact[:, 20:], bound[:, 20:]) > DO.C_HEAD


def test_slip_dropped_last_row():
    zz, g = _zz(37, 100, 5)
    out, t, _ = k_scaled_fwd(zz, 100)
    out[-1] = 0.0
    f = DO.scaled_fwd_bound(zz, 100)
    assert _ratio(out, f["out"], f["out_bound"]) > DO.C_HEAD
    d = k_scaled_bwd(g, zz, 100, torch.bfloat16)
    d[-1] = 0
    exact, bound = DO.scaled_bwd_bound(g, zz, 100, EB.U)
    assert _ratio(d, exact, bound) > DO.C_HEAD
    # FixedScaledDecoder: D summed without the last row
    T = torch.rand(10000, generator=torch.Generator().manual_seed(2)) * 3e-4
    _, S, _, _ = k_fixed(g[:-1], zz[:-1, :100], T, F32)
    b = DO.fixed_bwd_bound(g, zz[:, :100], S, EB.U32)
    dT_short = -(g[:-1].double() * zz[:-1, :100].double()).sum() / S.double() ** 2
    assert _ratio(dT_short, b["dT"], b["dT_bound"]) > DO.C_HEAD


def test_slip_wrong_dT():
    zz, g = _zz(50, 8, 6)
    T = torch.rand(10000, generator=torch.Generator().manual_seed(3)) * 3e-4      # S near 1.5, not 1
    S = T.sum()
    b = DO.fixed_bwd_bound(g, zz[:, :8], S, EB.U32)
    D = (g.double() * zz[:, :8].double()).sum()
    for wrong in (-D / S.double(), D / S.double() ** 2):                # a missing square; the sign
        assert _ratio(wrong, b["dT"], b["dT_bound"]) > DO.C_HEAD
