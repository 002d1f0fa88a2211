"""The learned-temperature decoder heads on the GPU: the row kernels of csrc/scaled_head.cu against their per-element fp64
bounds, the whole heads against the vendored reference decoders.py in fp64, training through `train(decoder=...)`, the
reference's own ScaledDecoder under TransformerModel, and the data-parallel gradient bucket."""
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import decoders_oracle as DO, error_budget as EB
from transformerscandobayesianinference_b200 import _lib as L
from transformerscandobayesianinference_b200 import bar_distribution, decoders, encoders, engine, priors, transformer
from transformerscandobayesianinference_b200 import train as train_mod, utils

DTYPES = {"bf16": torch.bfloat16, "fp32": torch.float32}


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), device="cuda:0", dtype=dtype)


# ------------------------------------------------------------------------------------------------------------------
# row kernels alone
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("rows", [1, 13, 4099])
@pytest.mark.parametrize("n_out", [1, 2, 5, 100, 1000])
def test_scaled_row_kernels_within_bounds(cuda_device, n_out, rows, precision):
    gen = torch.Generator(device=cuda_device).manual_seed(n_out * 7 + rows)
    nz = n_out + 10
    zz = torch.randn(rows, nz + 3, device=cuda_device, generator=gen)[:, :nz]        # a pitch that is not nz
    zz[:, n_out:] *= 4
    g = torch.randn(rows, n_out, device=cuda_device, generator=gen)
    out, temp = _nan(rows, n_out + 1)[:, :n_out], _nan(rows)
    L.scaled_head_fwd(zz, n_out, out, temp)
    f = DO.scaled_fwd_bound(zz, n_out)
    EB.check(f"scaled out n={n_out} rows={rows}", out, f["out"], f["out_bound"], DO.C_HEAD)
    EB.check(f"scaled temp n={n_out} rows={rows}", temp, f["temp"], f["temp_bound"], DO.C_HEAD)
    dt = DTYPES[precision]
    pad = (nz + 7) // 8 * 8
    dzz = _nan(rows, pad, dtype=dt)
    L.scaled_head_bwd(g, zz, temp, n_out, dzz, pad)
    exact, bound = DO.scaled_bwd_bound(g, zz, n_out, EB.U if dt == torch.bfloat16 else EB.U32)
    EB.check(f"scaled dzz n={n_out} rows={rows} {precision}", dzz[:, :nz], exact, bound, DO.C_HEAD)
    assert (dzz[:, nz:] == 0).all()


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("rows", [1, 13, 4099])
@pytest.mark.parametrize("n_out", [1, 2, 5, 100, 1000])
def test_fixed_row_kernels_within_bounds(cuda_device, n_out, rows, precision):
    gen = torch.Generator(device=cuda_device).manual_seed(n_out * 5 + rows)
    z = torch.randn(rows, n_out, device=cuda_device, generator=gen)
    g = torch.randn(rows, n_out, device=cuda_device, generator=gen)
    T = torch.rand(10000, device=cuda_device, generator=gen) * 3e-4
    out, S = _nan(rows, n_out), _nan(1)
    L.fixed_scaled_head_fwd(z, n_out, T, out, S)
    f = DO.fixed_fwd_bound(z, T)
    EB.check(f"fixed out n={n_out} rows={rows}", out, f["out"], f["out_bound"], DO.C_HEAD)
    EB.check(f"fixed S n={n_out} rows={rows}", S[0], f["S"], f["S_bound"], DO.C_HEAD)
    dt = DTYPES[precision]
    pad = (n_out + 7) // 8 * 8
    dz, dT = _nan(rows, pad, dtype=dt), _nan(10000)
    L.fixed_scaled_head_bwd(g, z, S, n_out, dz, dT, pad)
    b = DO.fixed_bwd_bound(g, z, S, EB.U if dt == torch.bfloat16 else EB.U32)
    EB.check(f"fixed dz n={n_out} rows={rows} {precision}", dz[:, :n_out], b["dz"], b["dz_bound"], DO.C_HEAD)
    EB.check(f"fixed dT n={n_out} rows={rows} {precision}", dT, b["dT"].expand(10000), b["dT_bound"].expand(10000), DO.C_HEAD)
    assert (dz[:, n_out:] == 0).all() and torch.equal(dT, dT[:1].expand(10000))


def test_row_kernels_are_deterministic(cuda_device):
    zz = torch.randn(3000, 110, device=cuda_device)
    g = torch.randn(3000, 100, device=cuda_device)
    T = torch.rand(10000, device=cuda_device)
    runs = []
    for _ in range(2):
        out, temp, dzz = torch.empty(3000, 100, device=cuda_device), torch.empty(3000, device=cuda_device), \
            torch.empty(3000, 112, device=cuda_device, dtype=torch.bfloat16)
        L.scaled_head_fwd(zz, 100, out, temp)
        L.scaled_head_bwd(g, zz, temp, 100, dzz, 112)
        S, dz, dT = torch.empty(1, device=cuda_device), torch.empty(3000, 104, device=cuda_device), \
            torch.empty(10000, device=cuda_device)
        fout = torch.empty(3000, 100, device=cuda_device)
        L.fixed_scaled_head_fwd(zz[:, :100], 100, T, fout, S)
        L.fixed_scaled_head_bwd(g, zz[:, :100], S, 100, dz, dT, 104)
        runs.append((out, temp, dzz, fout, S, dz, dT))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------------------
# whole heads against the vendored reference in fp64
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref():
    mod = DO.load_reference()
    if mod is None:
        pytest.skip("oracle/_ref has not been built (python oracle/build_ref.py)")
    return mod


def _run_head(m, hq, precision):
    hq = hq.detach().clone().requires_grad_()
    out = m.fused(hq, (hq.shape[0],), precision)
    gout = torch.randn_like(out)
    out.backward(gout)
    return out.detach(), gout, hq.grad


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("n_out", [1, 100, 1000])
def test_scaled_head_matches_reference_fp64(cuda_device, ref, monkeypatch, precision, n_out):
    monkeypatch.setattr(random, "random", lambda: 0.0)
    torch.manual_seed(n_out)
    E, nhid, Nq = 256, 512, 1000
    m = decoders.ScaledDecoder(E, nhid, n_out).to(cuda_device)
    with torch.no_grad():
        m.linear2.weight.mul_(8)
    hq = torch.randn(Nq, E, device=cuda_device).to(DTYPES[precision])
    out, gout, dhq = _run_head(m, hq, precision)
    r = DO.scaled_head(hq, m.linear.weight, m.linear.bias, m.linear1.weight, m.linear1.bias, m.linear2.weight,
                       m.linear2.bias, gout)
    # the unmodified reference module in fp64 on the same weights (its constants are float32, as in the kernel)
    rm = ref.ScaledDecoder(E, nhid, n_out).to(cuda_device).double()
    rm.load_state_dict(m.state_dict())
    # (its temperature constants are a float32 tensor, which an fp64 module cannot multiply: the host tests hold the
    # restatement's temperature division to the reference module run with float64 as torch's default dtype)
    with torch.no_grad():
        rz = rm.linear1(torch.nn.GELU()(rm.linear(hq.double())))
    torch.testing.assert_close(rz, r["zz"][:, :n_out], rtol=1e-12, atol=1e-12)
    u = EB.U if precision == "bf16" else EB.U32
    W12 = torch.cat([m.linear1.weight, m.linear2.weight])
    b12 = torch.cat([m.linear1.bias, m.linear2.bias])
    bd = DO.head_bounds(r, hq, m.linear.weight, m.linear.bias, W12, b12, u, True, n_out, gout)
    tag = f"scaled n={n_out} {precision}"
    EB.check(f"{tag} logits", out, r["out"], bd["out"], DO.C_HEAD_WHOLE)
    EB.check(f"{tag} dhq", dhq, r["dhq"], bd["dhq"], DO.C_HEAD_WHOLE)
    EB.check(f"{tag} linear.weight", m.linear.weight.grad, r["dW"], bd["dW"], DO.C_HEAD_WHOLE)
    EB.check(f"{tag} linear.bias", m.linear.bias.grad, r["db"], bd["db"], DO.C_HEAD_WHOLE)
    dW12 = torch.cat([m.linear1.weight.grad, m.linear2.weight.grad])
    db12 = torch.cat([m.linear1.bias.grad, m.linear2.bias.grad])
    EB.check(f"{tag} linear1/2.weight", dW12, r["dW12"], bd["dW2"], DO.C_HEAD_WHOLE)
    EB.check(f"{tag} linear1/2.bias", db12, r["db12"], bd["db2"], DO.C_HEAD_WHOLE)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("n_out", [1, 100, 1000])
def test_fixed_head_matches_reference_fp64(cuda_device, ref, precision, n_out):
    torch.manual_seed(n_out + 1)
    E, nhid, Nq = 256, 512, 1000
    m = decoders.FixedScaledDecoder(E, nhid, n_out).to(cuda_device)
    with torch.no_grad():
        m.T.uniform_(0, 3e-4)
    hq = torch.randn(Nq, E, device=cuda_device).to(DTYPES[precision])
    out, gout, dhq = _run_head(m, hq, precision)
    rm = ref.FixedScaledDecoder(E, nhid, n_out).to(cuda_device).double()
    rm.load_state_dict(m.state_dict())
    x = hq.double().requires_grad_()
    rout = rm(x)
    rout.backward(gout.double())
    r = DO.fixed_head(hq, m.mapper[0].weight, m.mapper[0].bias, m.mapper[2].weight, m.mapper[2].bias, m.T, gout)
    torch.testing.assert_close(rout.detach(), r["out"], rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(rm.T.grad, r["dT"], rtol=1e-10, atol=0)
    u = EB.U if precision == "bf16" else EB.U32
    bd = DO.head_bounds(r, hq, m.mapper[0].weight, m.mapper[0].bias, m.mapper[2].weight, m.mapper[2].bias, u, False,
                        n_out, gout)
    tag = f"fixed n={n_out} {precision}"
    EB.check(f"{tag} logits", out, r["out"], bd["out"], DO.C_HEAD_WHOLE)
    EB.check(f"{tag} dhq", dhq, r["dhq"], bd["dhq"], DO.C_HEAD_WHOLE)
    EB.check(f"{tag} mapper.0.weight", m.mapper[0].weight.grad, r["dW0"], bd["dW"], DO.C_HEAD_WHOLE)
    EB.check(f"{tag} mapper.0.bias", m.mapper[0].bias.grad, r["db0"], bd["db"], DO.C_HEAD_WHOLE)
    EB.check(f"{tag} mapper.2.weight", m.mapper[2].weight.grad, r["dW2"], bd["dW2"], DO.C_HEAD_WHOLE)
    EB.check(f"{tag} mapper.2.bias", m.mapper[2].bias.grad, r["db2"], bd["db2"], DO.C_HEAD_WHOLE)
    EB.check(f"{tag} T", m.T.grad, r["dT"], bd["dT"].expand(10000), DO.C_HEAD_WHOLE)
    assert torch.equal(m.T.grad, m.T.grad[:1].expand(10000))


def test_direct_call_any_leading_shape(cuda_device, monkeypatch):
    draws = []
    monkeypatch.setattr(random, "random", lambda: draws.append(1) or 0.0)
    torch.manual_seed(0)
    for cls in (decoders.ScaledDecoder, decoders.FixedScaledDecoder):
        m = cls(64, 96, 7).to(cuda_device)
        x = torch.randn(5, 3, 2, 64, device=cuda_device)
        out = m(x)
        assert out.shape == (5, 3, 2, 7) and out.dtype == torch.float32 and torch.isfinite(out).all()
        flat = m(x.reshape(-1, 64))
        torch.testing.assert_close(out.reshape(-1, 7), flat, rtol=0, atol=0)
    assert len(draws) == 2          # ScaledDecoder: one draw per forward; FixedScaledDecoder: none


# ------------------------------------------------------------------------------------------------------------------
# under TransformerModel and train()
# ------------------------------------------------------------------------------------------------------------------
def _model(decoder, dev, E=128, n_out=20):
    torch.manual_seed(0)
    m = transformer.TransformerModel(encoders.Linear(1, E), n_out, E, 1, 2 * E, 1, 0.0, y_encoder=encoders.Linear(1, E),
                                     decoder=decoder).to(dev)
    return m


def test_reference_scaled_decoder_runs_under_transformer_model(cuda_device, ref, monkeypatch, capsys):
    """The reference's own class is a custom decoder: it runs as torch ops on the [T - sep, B, E] query rows, so its
    print of temps[:, :2] no longer raises."""
    monkeypatch.setattr(random, "random", lambda: 0.995)
    m = _model(ref.ScaledDecoder, cuda_device)
    x, y = torch.rand(12, 4, 1, device=cuda_device), torch.randn(12, 4, device=cuda_device)
    out = m((x, y), single_eval_pos=8)
    assert out.shape == (4, 4, 20) and torch.isfinite(out).all()
    assert "torch.Size([4, 4])" in capsys.readouterr().out
    out.sum().backward()
    assert m.decoder.linear2.weight.grad is not None


@pytest.mark.parametrize("cls", ["ScaledDecoder", "FixedScaledDecoder"])
def test_transformer_model_routes_package_heads_to_the_fused_path(cuda_device, monkeypatch, capsys, cls):
    draws = []
    monkeypatch.setattr(random, "random", lambda: draws.append(1) or 0.995)
    m = _model(getattr(decoders, cls), cuda_device)
    calls = []
    fn = engine.ScaledDecoderFn if cls == "ScaledDecoder" else engine.FixedScaledDecoderFn
    orig = fn.apply
    monkeypatch.setattr(fn, "apply", lambda *a: calls.append(1) or orig(*a))
    x, y = torch.rand(12, 4, 1, device=cuda_device), torch.randn(12, 4, device=cuda_device)
    out = m((x, y), single_eval_pos=8)
    assert out.shape == (4, 4, 20) and torch.isfinite(out).all() and calls == [1]
    if cls == "ScaledDecoder":
        assert draws == [1] and capsys.readouterr().out.startswith("torch.Size([4, 4])")
    else:
        assert draws == []


@pytest.mark.parametrize("cls", ["ScaledDecoder", "FixedScaledDecoder"])
def test_train_with_head_is_finite_and_learns(cuda_device, cls):
    torch.manual_seed(0); random.seed(0)
    ys = priors.fast_gp.get_batch(500, 30, 1, device="cuda:0")[1]
    crit = bar_distribution.FullSupportBarDistribution(bar_distribution.get_bucket_limits(100, ys=ys.cpu()))
    kw = dict(criterion=crit, encoder_generator=encoders.Linear, emsize=128, nhid=256, nlayers=2, nhead=4, dropout=0.0,
              epochs=6, steps_per_epoch=20, batch_size=16, bptt=30, lr=3e-3, warmup_epochs=1,
              y_encoder_generator=encoders.Linear, decoder=getattr(decoders, cls),
              extra_prior_kwargs_dict={"num_features": 1, "hyperparameters": {"noise": .1, "outputscale": .1, "lengthscale": .1}},
              single_eval_pos_gen=utils.get_weighted_single_eval_pos_sampler(30), verbose=False)
    total_loss, _, model = train_mod.train(priors.fast_gp.DataLoader, **kw)
    assert total_loss == total_loss and abs(total_loss) < float("inf")
    assert all(torch.isfinite(p).all() for p in model.parameters())
    kw.update(epochs=1, steps_per_epoch=4, warmup_epochs=0, lr=0.0)
    torch.manual_seed(0); random.seed(0)
    first_loss, _, _ = train_mod.train(priors.fast_gp.DataLoader, **kw)
    assert total_loss < first_loss - 0.02, (first_loss, total_loss)


@pytest.mark.parametrize("cls,n_grads", [("ScaledDecoder", 6), ("FixedScaledDecoder", 5)])
def test_head_gradients_form_one_bucket(cuda_device, monkeypatch, cls, n_grads):
    buckets = []
    monkeypatch.setattr(engine, "GRAD_BUCKET_HOOK", lambda flat: buckets.append(flat.clone()))
    monkeypatch.setattr(engine, "GRAD_BUCKET_SYNC", lambda: None)
    monkeypatch.setattr(random, "random", lambda: 0.0)
    m = _model(getattr(decoders, cls), cuda_device)
    x, y = torch.rand(12, 4, 1, device=cuda_device), torch.randn(12, 4, device=cuda_device)
    m((x, y), single_eval_pos=8).square().mean().backward()
    torch.cuda.synchronize()
    head = list(m.decoder.parameters())
    assert len(head) == n_grads and len(buckets) == 1 + len(m.transformer_encoder.layers)
    got = buckets[0]
    assert got.numel() == sum(p.numel() for p in head)
    assert torch.equal(got.sort().values, torch.cat([p.grad.flatten() for p in head]).sort().values)
