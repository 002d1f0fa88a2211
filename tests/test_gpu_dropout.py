"""Training-mode dropout (reference train.py:22 default 0.2; tabular checkpoints 0.5): the engine's counter-based masks at
the reference layer's four sites, checked against an fp64 oracle that consumes EXACTLY the masks the kernels use
(pfn_dropout_keep_mask), plus the statistics of the mask generator."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L, bar_distribution, encoders, engine, transformer
from oracle import error_budget as EB, pfn_oracle as O


def test_keep_mask_statistics_and_elementwise_kernel(cuda_device):
    dev = cuda_device
    for p in (0.2, 0.5):
        thr = L.drop_threshold(p)
        m = torch.empty(4096, 512, device=dev, dtype=torch.uint8)
        L.dropout_keep_mask(m, 1234, thr)
        keep = m.float()
        assert abs(keep.mean().item() - (1 - thr / 256)) < 2e-3
        assert abs(keep.mean(0).std().item()) < 0.02 and abs(keep.mean(1).std().item()) < 0.05       # no row / column structure
        m2 = torch.empty_like(m)
        L.dropout_keep_mask(m2, 1235, thr)
        agree = (m == m2).float().mean().item()
        assert abs(agree - ((1 - thr / 256) ** 2 + (thr / 256) ** 2)) < 5e-3                            # seeds are independent
        for dt in (torch.float32, torch.bfloat16):
            x = torch.randn(4096, 512, device=dev).to(dt)
            r = torch.randn(4096, 512, device=dev).to(dt)
            u = EB.U32 if dt == torch.float32 else EB.U
            out = torch.empty_like(x)
            L.dropout(x, out, 1234, thr, residual=r)
            exact, bound = EB.dropout(x, m, thr, r, u)
            EB.check(f"dropout + residual p={p} {dt}", out, exact, bound, EB.C_DROPOUT)
            y = x.clone()
            L.dropout(y, y, 1234, thr)                                                                  # in place, no residual
            exact, bound = EB.dropout(x, m, thr, None, u)
            EB.check(f"dropout in place p={p} {dt}", y, exact, bound, EB.C_DROPOUT)


@pytest.mark.parametrize("p", [0.2, 0.5])
def test_training_step_with_dropout_matches_mask_consuming_oracle(cuda_device, p):
    dev = cuda_device
    T, B, F, E, H, nhid, NL, n_out, sep = 24, 3, 2, 64, 2, 128, 2, 12, 14
    torch.manual_seed(17)
    m = transformer.TransformerModel(encoders.Linear(F, E), n_out, E, H, nhid, NL, p, y_encoder=encoders.Linear(1, E)).to(dev)
    with torch.no_grad():
        for l in m.transformer_encoder.layers:
            l.linear2.weight.normal_(0, 0.05); l.self_attn.out_proj.weight.normal_(0, 0.05)
    m.precision = "fp32"
    m.train()
    x, y = torch.rand(T, B, F, device=dev), torch.randn(T, B, device=dev).clamp(-2.5, 2.5)
    crit = bar_distribution.FullSupportBarDistribution(torch.linspace(-3, 3, n_out + 1)).to(dev)
    torch.manual_seed(99)
    seed = int(torch.randint(0, 2 ** 31 - 1, (1,)).item())        # what TransformerModel.forward will draw
    torch.manual_seed(99)
    logits = m((x, y), single_eval_pos=sep)
    loss = crit(logits.reshape(-1, n_out), y[sep:].flatten()).mean()
    loss.backward()
    # eval mode is deterministic and differs from the training-mode output
    m.eval()
    with torch.no_grad():
        assert not torch.allclose(m((x, y), single_eval_pos=sep), logits)
    m.train()

    thr = L.drop_threshold(p)
    scale = 256.0 / (256 - thr)

    def mask(rows, cols, li, site):
        out = torch.empty(rows, cols, device=dev, dtype=torch.uint8)
        L.dropout_keep_mask(out, engine.site_seed(seed, li, site), thr)
        return out.cpu().double()
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    P = O.params_from_state_dict(sd, NL, torch.float64)
    leaves = {}
    for i, lp in enumerate(P["layers"]):
        pre = f"transformer_encoder.layers.{i}."
        leaves.update({pre + "self_attn.in_proj_weight": lp["in_w"], pre + "self_attn.in_proj_bias": lp["in_b"],
                       pre + "self_attn.out_proj.weight": lp["out_w"], pre + "self_attn.out_proj.bias": lp["out_b"],
                       pre + "linear1.weight": lp["w1"], pre + "linear1.bias": lp["b1"], pre + "linear2.weight": lp["w2"],
                       pre + "linear2.bias": lp["b2"], pre + "norm1.weight": lp["g1"], pre + "norm2.bias": lp["be2"]})
    leaves["encoder.weight"] = P["enc_w"]
    for t in leaves.values():
        t.requires_grad_(True)
    h = O.embed_ref(x.cpu().double(), y.cpu().double(), P["enc_w"], P["enc_b"], P["yenc_w"], P["yenc_b"], sep)
    for li, lp in enumerate(P["layers"]):
        keep = {"attn": mask(B * H * T, T, li, 0).reshape(B * H, T, T), "out": mask(T * B, E, li, 1),
                "gelu": mask(T * B, nhid, li, 2), "mlp": mask(T * B, E, li, 3)}
        h = O.encoder_layer_dropout_ref(h, lp, T, B, H, sep, keep, scale)
    ref_logits = O.gelu_erf(h[sep * B:] @ P["dec_w0"].T + P["dec_b0"]) @ P["dec_w2"].T + P["dec_b2"]
    ref = O.bar_nll_ref(ref_logits, y[sep:].flatten().cpu().double(), torch.linspace(-3, 3, n_out + 1).double(), True).mean()
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-4 * abs(ref.item()), (loss.item(), ref.item())
    named = dict(m.named_parameters())
    for k, t in leaves.items():
        got = named[k].grad.double().cpu()
        assert (got - t.grad).abs().max().item() <= 2e-3 * (t.grad.abs().max().item() + 1e-9), k


def test_default_train_arguments_run_with_dropout(cuda_device):
    """`train()` with the reference's default dropout = 0.2 (train.py:22) must run (it raised in round 1), bf16 engine."""
    from transformerscandobayesianinference_b200 import priors, train as train_mod, utils
    torch.manual_seed(0)
    ys = priors.fast_gp.get_batch(200, 20, 1, device="cuda:0")[1]
    crit = bar_distribution.FullSupportBarDistribution(bar_distribution.get_bucket_limits(50, ys=ys.cpu()))
    loss, pos, model = train_mod.train(priors.fast_gp.DataLoader, crit, encoders.Linear, emsize=256, nhid=256, nlayers=2, nhead=2,
                                       epochs=2, steps_per_epoch=4, batch_size=8, bptt=20, lr=1e-3, warmup_epochs=0,
                                       y_encoder_generator=encoders.Linear, extra_prior_kwargs_dict={"num_features": 1},
                                       single_eval_pos_gen=utils.get_weighted_single_eval_pos_sampler(20), verbose=False)
    assert loss == loss and model.dropout == 0.2


@pytest.mark.parametrize("T,B,H,sep,p", [(200, 2, 2, 100, 0.5), (384, 8, 4, 200, 0.2), (130, 1, 2, 0, 0.5), (256, 2, 1, 255, 0.2)])
def test_tcgen05_attention_with_probability_dropout(cuda_device, T, B, H, sep, p):
    """tensor-core forward / dQ / dK,dV kernels (bf16, head dim 128) with dropout on the probabilities vs the exact fp64
    attention that consumes the same keep mask, O = (softmax(S) m / (1-p)) V and its gradients, within the per-element
    bounds of oracle/error_budget.py."""
    dev = cuda_device
    torch.manual_seed(T + sep)
    dh, E = 128, H * 128
    thr, seed = L.drop_threshold(p), 424242 + T
    scale = 256.0 / (256 - thr)
    qkv = (torch.randn(T * B, 3 * E, device=dev) * 1.2).to(torch.bfloat16)
    out = torch.empty(T * B, E, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B * H, T, device=dev)
    L.attention_fwd(qkv, out, lse, T, B, H, dh, sep, use_tc=True, drop=(seed, thr))
    dout = torch.randn(T * B, E, device=dev).to(torch.bfloat16)
    dqkv = torch.full_like(qkv, float("nan"))
    delta = torch.empty_like(lse)
    L.attention_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, dh, sep, use_tc=True, drop=(seed, thr))
    torch.cuda.synchronize()
    keep = torch.empty(B * H * T, T, device=dev, dtype=torch.uint8)
    L.dropout_keep_mask(keep, seed, thr)
    torch.cuda.synchronize()
    assert torch.isfinite(dqkv.float()).all()
    f = EB.attention_fwd(qkv, T, B, H, dh, sep, EB.U, keep.reshape(B, H, T, T), scale)
    EB.check_attention_fwd(out, lse, f, EB.C_ATT_OUT, EB.C_ATT_LSE)
    EB.check_attention_bwd(dqkv, EB.attention_bwd(f, dout, out), EB.C_ATT_GRAD)
    # the fp32-FMA kernels draw the same mask: same outputs up to bf16 rounding
    out2 = torch.empty_like(out); lse2 = torch.empty_like(lse)
    L.attention_fwd(qkv, out2, lse2, T, B, H, dh, sep, use_tc=False, drop=(seed, thr))
    assert (out2.float() - out.float()).abs().max().item() <= 3e-2 * out.float().abs().max().item()


def test_bf16_engine_training_step_with_dropout_on_tensor_cores(cuda_device):
    """Whole bf16 step (wgmma GEMMs + tensor-core attention, head dim 128) with dropout 0.5: loss within 1e-2 of the
    mask-consuming fp64 oracle, gradient norms within 8 %."""
    dev = cuda_device
    T, B, F, E, H, nhid, NL, n_out, sep, p = 160, 4, 1, 256, 2, 512, 2, 20, 96, 0.5
    torch.manual_seed(23)
    m = transformer.TransformerModel(encoders.Linear(F, E), n_out, E, H, nhid, NL, p, y_encoder=encoders.Linear(1, E)).to(dev)
    with torch.no_grad():
        for l in m.transformer_encoder.layers:
            l.linear2.weight.normal_(0, 0.03); l.self_attn.out_proj.weight.normal_(0, 0.03)
    m.precision = "bf16"
    m.train()
    x, y = torch.rand(T, B, F, device=dev), torch.randn(T, B, device=dev).clamp(-2.5, 2.5)
    crit = bar_distribution.FullSupportBarDistribution(torch.linspace(-3, 3, n_out + 1)).to(dev)
    torch.manual_seed(5)
    seed = int(torch.randint(0, 2 ** 31 - 1, (1,)).item())
    torch.manual_seed(5)
    loss = crit(m((x, y), single_eval_pos=sep).reshape(-1, n_out), y[sep:].flatten()).mean()
    loss.backward()
    thr = L.drop_threshold(p)
    scale = 256.0 / (256 - thr)

    def mask(rows, cols, li, site):
        out = torch.empty(rows, cols, device=dev, dtype=torch.uint8)
        L.dropout_keep_mask(out, engine.site_seed(seed, li, site), thr)
        return out.cpu().double()
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    P = O.params_from_state_dict(sd, NL, torch.float64)
    leaves = {f"transformer_encoder.layers.{i}.linear1.weight": lp["w1"] for i, lp in enumerate(P["layers"])}
    leaves.update({f"transformer_encoder.layers.{i}.self_attn.in_proj_weight": lp["in_w"] for i, lp in enumerate(P["layers"])})
    for t in leaves.values():
        t.requires_grad_(True)
    h = O.embed_ref(x.cpu().double(), y.cpu().double(), P["enc_w"], P["enc_b"], P["yenc_w"], P["yenc_b"], sep)
    for li, lp in enumerate(P["layers"]):
        keep = {"attn": mask(B * H * T, T, li, 0).reshape(B * H, T, T), "out": mask(T * B, E, li, 1),
                "gelu": mask(T * B, nhid, li, 2), "mlp": mask(T * B, E, li, 3)}
        h = O.encoder_layer_dropout_ref(h, lp, T, B, H, sep, keep, scale)
    ref_logits = O.gelu_erf(h[sep * B:] @ P["dec_w0"].T + P["dec_b0"]) @ P["dec_w2"].T + P["dec_b2"]
    ref = O.bar_nll_ref(ref_logits, y[sep:].flatten().cpu().double(), torch.linspace(-3, 3, n_out + 1).double(), True).mean()
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-2 * abs(ref.item()), (loss.item(), ref.item())
    named = dict(m.named_parameters())
    for k, t in leaves.items():
        a, b = named[k].grad.double().cpu().norm().item(), t.grad.norm().item()
        assert abs(a - b) <= 8e-2 * b, (k, a, b)
