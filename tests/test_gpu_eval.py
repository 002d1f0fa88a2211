"""Inference / evaluation path on the GPU: BarDistribution helpers on device tensors
against the reference goldens, DataLoader.validate, the exact-GP baseline `fast_gp.evaluate`, and the other heads /
encoders (BCE, CE + class-embedding y-encoder, positional encodings, wide feature encoder) through the CUDA stack."""
import os

import pytest
import torch
from torch import nn

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import bar_distribution, encoders, positional_encodings, priors, transformer
from transformerscandobayesianinference_b200 import train as train_mod
from oracle import pfn_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("n_bars", [7, 100, 1000])
def test_bar_distribution_helpers_on_device_match_reference(cuda_device, n_bars):
    """mean / mode / quantile / ei / forward on CUDA tensors vs outputs of the unmodified reference (tests/golden/bar.pt;
    reference bar_distribution.py:25-80, 89-117)."""
    e = torch.load(os.path.join(GOLD, "bar.pt"))[n_bars]
    dev = cuda_device
    bd = bar_distribution.BarDistribution(e["borders"]).to(dev)
    lg = e["logits"].to(dev)
    assert torch.equal(bd.map_to_bucket_idx(e["y"].to(dev)).cpu(), e["idx"])
    assert torch.allclose(bd(lg, e["y"].to(dev)).cpu(), e["nll"], rtol=1e-5, atol=1e-5)
    assert torch.allclose(bd.mean(lg).cpu(), e["mean"], rtol=1e-5, atol=1e-5)
    assert torch.allclose(bd.mode(lg).cpu(), e["mode"])
    assert torch.allclose(bd.quantile(lg).cpu(), e["quantile"], rtol=1e-4, atol=1e-4)
    assert torch.allclose(bd.ei(lg, 0.3, maximize=True).cpu(), e["ei_max"], rtol=1e-5, atol=1e-5)
    assert torch.allclose(bd.ei(lg, 0.3, maximize=False).cpu(), e["ei_min"], rtol=1e-5, atol=1e-5)
    fs = bar_distribution.FullSupportBarDistribution(e["borders"]).to(dev)
    assert torch.allclose(fs(lg, e["y_full"].to(dev)).cpu(), e["nll_full"], rtol=1e-5, atol=1e-5)
    assert torch.allclose(fs.mean(lg).cpu(), e["mean_full"], rtol=1e-5, atol=1e-5)


def _small_model(dev, n_out, F=1, E=64, y_encoder=None, encoder=None, pos=None, L=2):
    torch.manual_seed(3)
    m = transformer.TransformerModel(encoder or encoders.Linear(F, E), n_out, E, 2, 128, L, 0.0,
                                     y_encoder=y_encoder or encoders.Linear(1, E), pos_encoder=pos).to(dev)
    with torch.no_grad():
        for l in m.transformer_encoder.layers:
            l.linear2.weight.normal_(0, 0.05); l.self_attn.out_proj.weight.normal_(0, 0.05)
    m.precision = "fp32"
    return m


def test_fast_gp_mix_validate_matches_manual_loop(cuda_device):
    """DataLoader.validate (reference priors/fast_gp_mix.py:140-153): MSE of the bar mean at the first query row for every
    eval position, under no_grad / eval -- equal to a hand-rolled loop over the same batch, and leaves the model in train mode."""
    dev = cuda_device
    m = _small_model(dev, 20)
    m.criterion = bar_distribution.FullSupportBarDistribution(torch.linspace(-4, 4, 21)).to(dev)
    dl = priors.fast_gp_mix.DataLoader(num_steps=1, batch_size=8, seq_len=12, num_features=1, device="cuda:0",
                                       batch_size_per_gp_sample=4)
    torch.manual_seed(11)
    with torch.no_grad():
        got = dl.validate(m)
    assert got.shape == (12,) and torch.isfinite(got).all() and m.training
    torch.manual_seed(11)
    (x, y), t = dl.gbm(**dl.get_batch_kwargs, fuse_x_y=False)
    m.eval()
    with torch.no_grad():
        want = torch.stack([((m.criterion.mean(m((x, y), single_eval_pos=p))[0] - t[p]) ** 2).mean() for p in range(12)])
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-6)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items() if not k.startswith("criterion")}
    P = O.params_from_state_dict(sd, 2, torch.float64)
    ref_logits = O.transformer_forward_ref(P, x.cpu().double(), y.cpu().double(), 5, 2)
    ref_mean = O.bar_mean_ref(ref_logits, torch.linspace(-4, 4, 21).double(), full_support=True)
    assert abs(((ref_mean[0] - t[5].cpu().double()) ** 2).mean().item() - want[5].item()) <= 1e-4 * (want[5].item() + 1e-6)


@pytest.mark.parametrize("use_mse", [False, True])
def test_fast_gp_evaluate_matches_per_t_closed_form(cuda_device, use_mse):
    """priors.fast_gp.evaluate (one factor from the fused sampler kernel + one triangular solve) vs the fp64 per-t
    restatement of reference priors/fast_gp.py:95-116."""
    torch.manual_seed(5)
    hps = {"noise": 0.05, "outputscale": 1.2, "lengthscale": 0.3}
    x, y, _ = priors.fast_gp.get_batch(6, 40, 2, device="cuda:0", hyperparameters=hps)
    all_l, means, secs = priors.fast_gp.evaluate(x, y, y, use_mse=use_mse, hyperparameters=hps, device="cuda:0")
    ref = O.gp_exact_predictive_ref(x.cpu().double(), y.cpu().double(), 0.3, 1.2, 0.05, use_mse=use_mse)
    assert all_l.shape == (39, 6) and means.shape == (40,) and means[0] == 0
    assert (all_l.double() - ref).abs().max().item() <= 2e-3 * (ref.abs().max().item() + 1)
    assert torch.allclose(means[1:].double(), ref.mean(1), rtol=2e-3, atol=2e-3)
    # the gpytorch-free get_model shim answers the same question point by point (reference :25-32, 95-106)
    model, lik = priors.fast_gp.get_model(x[:10].transpose(0, 1), y[:10].transpose(0, 1), hps)
    pred = lik(model(x[10].unsqueeze(1)))
    nll10 = -pred.log_prob(y[10].unsqueeze(1))
    want = O.gp_exact_predictive_ref(x.cpu().double(), y.cpu().double(), 0.3, 1.2, 0.05)[9]
    assert torch.allclose(nll10.cpu().double(), want, rtol=1e-3, atol=1e-3)


def test_bce_and_ce_heads_and_class_embedding_encoder(cuda_device):
    """BASELINE config 3 (BCE on a binarised target, reference train.py:84-85) and config 5 shape (CE head n_out = 5, y-encoder
    = class embedding `encoders.get_Canonical`, F = 784 input features, T = 6, single_eval_pos 5; reference train.py:86-88,
    encoders.py:22-33) through train.Trainer.step -- loss and input-layer gradients against the fp64 oracle."""
    dev = cuda_device
    torch.manual_seed(9)
    # ---- cfg 5 shape: 5-way 1-shot, CE head
    T, B, F, E, sep = 6, 16, 784, 64, 5
    m = _small_model(dev, 5, F=F, E=E, y_encoder=encoders.get_Canonical(5)(1, E))
    x = torch.rand(T, B, F, device=dev)
    ycls = torch.randint(0, 5, (T, B), device=dev)
    out = m((x, ycls), single_eval_pos=sep)
    assert out.shape == (1, B, 5)
    loss = nn.CrossEntropyLoss(reduction='none')(out.reshape(-1, 5), ycls[sep:].flatten()).mean()
    loss.backward()
    # oracle: embed by hand (encoder Linear + class embedding on the training rows), then the oracle's encoder stack
    sd = {k: v.detach().cpu().double() for k, v in m.state_dict().items()}
    xs = x.cpu().double() @ sd["encoder.weight"].T + sd["encoder.bias"]
    ys = sd["y_encoder.weight"][ycls.cpu()]                               # [T,B,E] (one feature: the embedding itself)
    h = torch.cat([xs[:sep] + ys[:sep], xs[sep:]], 0).reshape(T * B, E)
    for i in range(2):
        pre = f"transformer_encoder.layers.{i}."
        lp = {"in_w": sd[pre + "self_attn.in_proj_weight"], "in_b": sd[pre + "self_attn.in_proj_bias"],
              "out_w": sd[pre + "self_attn.out_proj.weight"], "out_b": sd[pre + "self_attn.out_proj.bias"],
              "w1": sd[pre + "linear1.weight"], "b1": sd[pre + "linear1.bias"], "w2": sd[pre + "linear2.weight"],
              "b2": sd[pre + "linear2.bias"], "g1": sd[pre + "norm1.weight"], "be1": sd[pre + "norm1.bias"],
              "g2": sd[pre + "norm2.weight"], "be2": sd[pre + "norm2.bias"]}
        h = O.encoder_layer_ref(h, lp, T, B, 2, sep)
    logits = O.gelu_erf(h[sep * B:] @ sd["decoder.0.weight"].T + sd["decoder.0.bias"]) @ sd["decoder.2.weight"].T + sd["decoder.2.bias"]
    ref = nn.CrossEntropyLoss()(logits, ycls[sep:].flatten().cpu())
    assert abs(loss.item() - ref.item()) <= 1e-4 * abs(ref.item())
    assert m.y_encoder.weight.grad.abs().sum() > 0 and m.encoder.weight.grad.abs().sum() > 0

    # ---- cfg 3 head: BCE through the Trainer's criterion dispatch (targets = binarised y)
    class TwoClass(priors.ridge.DataLoader):
        pass
    tr = train_mod.build_trainer(priors.ridge.DataLoader, nn.BCEWithLogitsLoss(reduction='none'), encoders.Linear, emsize=64, nhid=128,
                                 nlayers=2, nhead=2, dropout=0.0, epochs=1, steps_per_epoch=1, batch_size=8, bptt=20, lr=1e-3,
                                 warmup_epochs=0, y_encoder_generator=encoders.Linear,
                                 extra_prior_kwargs_dict=dict(num_features=18, device="cuda:0"), single_eval_pos_gen=10)
    tr.model.precision = "fp32"
    xb, yb = torch.rand(20, 8, 18, device=dev), (torch.rand(20, 8, device=dev) > 0.5).float()
    loss, losses = tr.step((xb, yb), yb, 10)
    assert losses.shape == (10, 8) and torch.isfinite(loss)


def test_positional_encoding_and_seqbn_paths(cuda_device):
    """Non-fused embedding variants (reference positional_encodings.py:21-49, utils.py:76-86 SeqBN via input_normalization)
    run in front of the CUDA encoder stack and back-propagate into their own parameters."""
    dev = cuda_device
    for pos in (positional_encodings.PositionalEncoding(64, 50), positional_encodings.LearnedPositionalEncoding(64, 50)):
        m = _small_model(dev, 3, F=2, pos=pos)
        x, y = torch.rand(9, 4, 2, device=dev), torch.randn(9, 4, device=dev)
        out = m((x, y), single_eval_pos=4)
        out.square().mean().backward()
        assert out.shape == (5, 4, 3) and torch.isfinite(out).all()
        if any(True for _ in pos.parameters()):
            assert all(p.grad is not None and p.grad.abs().sum() > 0 for p in pos.parameters())
    torch.manual_seed(1)
    m = transformer.TransformerModel(encoders.Linear(2, 64), 3, 64, 2, 128, 1, 0.0, y_encoder=encoders.Linear(1, 64),
                                     input_normalization=True).to(dev)
    m.precision = "fp32"
    out = m((torch.rand(9, 4, 2, device=dev), torch.randn(9, 4, device=dev)), single_eval_pos=4)
    out.square().mean().backward()
    assert m.input_ln.bn.weight.grad is not None


def test_explicit_reference_mask_takes_the_same_path(cuda_device):
    """reference transformer.py:60-65: passing the mask the reference would build itself changes nothing."""
    m = _small_model(cuda_device, 10).eval()
    torch.manual_seed(5)
    x, y = torch.rand(20, 3, 1, device=cuda_device), torch.rand(20, 3, device=cuda_device)
    with torch.no_grad():
        a = m((x, y), single_eval_pos=12)
        b = m((x, y), src_mask=m.generate_D_q_matrix(20, 8).to(cuda_device), single_eval_pos=12)
        with pytest.raises(NotImplementedError):
            m((x, y), src_mask=m.generate_square_subsequent_mask(20).to(cuda_device), single_eval_pos=12)
    assert torch.equal(a, b)
