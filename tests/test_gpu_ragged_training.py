"""Training with one single_eval_pos per dataset on the GPU: the ragged attention forward (with lse) and backward and the
ragged embedding against the fp64 oracle and against the scalar kernels dataset by dataset, the ragged `forward` and its
masked loss, and `train()` with `utils.per_dataset_sampler`."""
import os
import random
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import (_lib as L, _lib_ragged_train as LRT, bar_distribution, encoders,
                                                     priors, train as train_mod, utils)
from transformerscandobayesianinference_b200.transformer import TransformerModel
from oracle import error_budget as EB, pfn_oracle as O


def _ragged_attention(qkv, dout, T, B, H, dh, seps, use_tc, drop=None):
    dev = qkv.device
    n_keys = torch.tensor(seps, dtype=torch.int32, device=dev)
    out = torch.empty(T * B, H * dh, device=dev, dtype=qkv.dtype)
    lse = torch.empty(B * H, T, device=dev)
    LRT.attention_ragged_train_fwd(qkv, out, lse, T, B, H, dh, max(seps), n_keys, use_tc=use_tc, drop=drop)
    dqkv = torch.full_like(qkv, float("nan"))
    delta = torch.empty(B * H, T, device=dev)
    LRT.attention_ragged_train_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, dh, max(seps), n_keys, use_tc=use_tc,
                                   drop=drop)
    return out, lse, dqkv


def _scalar_attention(qkv, dout, T, B, H, dh, sep, use_tc, drop=None):
    dev = qkv.device
    out = torch.empty(T * B, H * dh, device=dev, dtype=qkv.dtype)
    lse = torch.empty(B * H, T, device=dev)
    L.attention_fwd(qkv, out, lse, T, B, H, dh, sep, use_tc=use_tc, drop=drop)
    dqkv = torch.full_like(qkv, float("nan"))
    delta = torch.empty(B * H, T, device=dev)
    L.attention_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, dh, sep, use_tc=use_tc, drop=drop)
    return out, lse, dqkv


def _columns(t, T, B, b):
    """Token rows of dataset b of a [T*B, cols] tensor."""
    return t.view(T, B, -1)[:, b]


# (T, B, H, separators): 0 and T in one batch; values that are not multiples of 64 or 128 with T not a multiple of 128;
# one dataset per distinct value with enough (batch, head) units for several waves of the persistent kernels
RAGGED_CASES = [
    (200, 4, 2, [0, 200, 77, 130]),
    (333, 5, 2, [1, 63, 65, 129, 257]),
    (300, 40, 4, [7 * b + 3 for b in range(40)]),
]


@pytest.mark.parametrize("use_tc,dh,dtype", [(True, 128, torch.bfloat16), (False, 64, torch.float32)])
@pytest.mark.parametrize("T,B,H,seps", RAGGED_CASES)
def test_ragged_attention_matches_oracle_and_scalar_kernels(cuda_device, use_tc, dh, dtype, T, B, H, seps):
    torch.manual_seed(T + B)
    E = H * dh
    qkv = (torch.randn(T * B, 3 * E, device=cuda_device) * 1.2).to(dtype)
    dout = torch.randn(T * B, E, device=cuda_device).to(dtype)
    out, lse, dqkv = _ragged_attention(qkv, dout, T, B, H, dh, seps, use_tc)
    torch.cuda.synchronize()
    assert torch.isfinite(dqkv.float()).all(), "dqkv not fully written"
    # each dataset gets what the scalar kernels give it at its own separator, bit for bit
    for s in sorted(set(seps)):
        o_s, l_s, d_s = _scalar_attention(qkv, dout, T, B, H, dh, s, use_tc)
        for b in (b for b in range(B) if seps[b] == s):
            assert torch.equal(_columns(out, T, B, b), _columns(o_s, T, B, b)), (s, b)
            assert torch.equal(lse.view(B, H, T)[b], l_s.view(B, H, T)[b]), (s, b)
            assert torch.equal(_columns(dqkv, T, B, b), _columns(d_s, T, B, b)), (s, b)
    if not use_tc and T > 256:
        return      # the fp32 dK bound does not model the kernel's serial fp32 sum over hundreds of query rows
    u = EB.U if dtype == torch.bfloat16 else EB.U32
    sep = torch.tensor(seps, device=cuda_device).view(B, 1, 1, 1)
    f = EB.attention_fwd(qkv, T, B, H, dh, sep, u)
    EB.check_attention_fwd(out, lse, f, EB.C_ATT_OUT, EB.C_ATT_LSE)
    EB.check_attention_bwd(dqkv, EB.attention_bwd(f, dout, out), EB.C_ATT_GRAD)


@pytest.mark.parametrize("use_tc,dh", [(True, 128), (False, 64)])
def test_ragged_attention_dropout_matches_scalar_kernels(cuda_device, use_tc, dh):
    T, B, H, seps = 150, 3, 2, [20, 150, 99]
    dtype = torch.bfloat16 if use_tc else torch.float32
    torch.manual_seed(5)
    E = H * dh
    qkv = torch.randn(T * B, 3 * E, device=cuda_device).to(dtype)
    dout = torch.randn(T * B, E, device=cuda_device).to(dtype)
    drop = (1234, L.drop_threshold(0.2))
    out, lse, dqkv = _ragged_attention(qkv, dout, T, B, H, dh, seps, use_tc, drop)
    for b, s in enumerate(seps):
        o_s, l_s, d_s = _scalar_attention(qkv, dout, T, B, H, dh, s, use_tc, drop)
        assert torch.equal(_columns(out, T, B, b), _columns(o_s, T, B, b)), b
        assert torch.equal(_columns(dqkv, T, B, b), _columns(d_s, T, B, b)), b


def test_ragged_attention_uniform_equals_scalar(cuda_device):
    T, B, H, dh = 260, 3, 2, 128
    torch.manual_seed(1)
    qkv = torch.randn(T * B, 3 * H * dh, device=cuda_device).to(torch.bfloat16)
    dout = torch.randn(T * B, H * dh, device=cuda_device).to(torch.bfloat16)
    got = _ragged_attention(qkv, dout, T, B, H, dh, [131] * B, True)
    want = _scalar_attention(qkv, dout, T, B, H, dh, 131, True)
    for g, w in zip(got, want):
        assert torch.equal(g, w)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_ragged_embedding(cuda_device, dtype):
    T, B, F, E = 37, 5, 3, 96
    seps = [0, 37, 5, 18, 36]
    torch.manual_seed(2)
    x, y = torch.randn(T * B, F, device=cuda_device), torch.randn(T * B, device=cuda_device)
    Wx, bx, wy, by = (torch.randn(*s, device=cuda_device) for s in ((E, F), (E,), (E,), (E,)))
    n_keys = torch.tensor(seps, dtype=torch.int32, device=cuda_device)
    out = torch.empty(T * B, E, device=cuda_device, dtype=dtype)
    LRT.embed_ragged_fwd(x, y, Wx, bx, wy, by, out, T, B, F, E, n_keys)
    dout = torch.randn(T * B, E, device=cuda_device).to(dtype)
    g = [torch.zeros(E, F, device=cuda_device)] + [torch.zeros(E, device=cuda_device) for _ in range(3)]
    LRT.embed_ragged_bwd(dout, x, y, *g, T, B, F, E, n_keys)
    train = (torch.arange(T, device=cuda_device).unsqueeze(1) < n_keys).reshape(-1, 1).double()
    want = x.double() @ Wx.double().T + bx.double() + train * (y.double().unsqueeze(1) * wy.double() + by.double())
    u = EB.U if dtype == torch.bfloat16 else EB.U32
    bound = (u + EB.U32 * (F + 2)) * (x.double().abs() @ Wx.double().abs().T + bx.double().abs()
                                      + train * (y.double().abs().unsqueeze(1) * wy.double().abs() + by.double().abs()))
    EB.check("ragged embed out", out, want, bound, 4.0)
    d = dout.double()
    depth = T * B
    for name, got, exact, mag in (
            ("dWx", g[0], d.T @ x.double(), d.abs().T @ x.double().abs()),
            ("dbx", g[1], d.sum(0), d.abs().sum(0)),
            ("dwy", g[2], (d * train * y.double().unsqueeze(1)).sum(0), (d.abs() * train * y.double().abs().unsqueeze(1)).sum(0)),
            ("dby", g[3], (d * train).sum(0), (d.abs() * train).sum(0))):
        EB.check(f"ragged embed {name}", got, exact, EB.U32 * depth * mag, 4.0)


# ---- the model --------------------------------------------------------------------------------------------------------
def _model(dev, emsize, nhead, precision, dropout=0.0, n_out=10):
    torch.manual_seed(0)
    m = TransformerModel(encoders.Linear(2, emsize), n_out, emsize, nhead, 2 * emsize, 2, dropout=dropout,
                         y_encoder=encoders.Linear(1, emsize))
    m.precision = precision
    return m.to(dev)


def _data(dev, T, B):
    g = torch.Generator().manual_seed(3)
    return torch.randn(T, B, 2, generator=g).to(dev), torch.randn(T, B, generator=g).to(dev)


def _grads(m):
    return {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("emsize,nhead,precision,dropout", [(256, 2, "bf16", 0.0), (128, 2, "fp32", 0.0),
                                                            (256, 2, "bf16", 0.2)])
def test_uniform_vector_is_the_scalar_call(cuda_device, emsize, nhead, precision, dropout):
    """B equal values run the scalar path: the same logits bit for bit, and the same gradients up to the order of the
    split-K weight-gradient reductions, which differs from one run of the scalar call to the next."""
    T, B, sep = 150, 4, 61
    m = _model(cuda_device, emsize, nhead, precision, dropout)
    m.train()
    x, y = _data(cuda_device, T, B)
    res = []
    for s in (sep, [sep] * B, torch.full((B,), sep, device=cuda_device)):
        m.zero_grad()
        torch.manual_seed(9)
        out = m((x, y), single_eval_pos=s)
        out.square().sum().backward()
        res.append((out.detach(), _grads(m)))
    for out, grads in res[1:]:
        assert torch.equal(out, res[0][0])
        assert grads.keys() == res[0][1].keys()
        for n in grads:
            ref = res[0][1][n]
            assert (grads[n] - ref).abs().max() <= 1e-5 * ref.abs().amax().clamp(min=1e-6), n


# per-element logit bound of tests/test_gpu_ragged_context.py, c * u * (|ref| + mean |ref|); per-tensor gradient bound of
# tests/test_gpu_model.py against the oracle (fp32: 2e-3 of the tensor's largest gradient; bf16: its 8 % probe bound)
C_MODEL = {"bf16": 16.0, "fp32": 512.0}
C_GRAD = {"bf16": 8e-2, "fp32": 2e-3}
UNIT = {"bf16": EB.U, "fp32": EB.U32}
BORDERS = torch.linspace(-3, 3, 21)


def _oracle_leaves(P):
    """The fp64 oracle parameters by the model's parameter names, each a leaf that requires grad."""
    leaves = {"encoder.weight": P["enc_w"], "encoder.bias": P["enc_b"], "y_encoder.weight": P["yenc_w"],
              "y_encoder.bias": P["yenc_b"], "decoder.0.weight": P["dec_w0"], "decoder.0.bias": P["dec_b0"],
              "decoder.2.weight": P["dec_w2"], "decoder.2.bias": P["dec_b2"]}
    names = {"in_w": "self_attn.in_proj_weight", "in_b": "self_attn.in_proj_bias", "out_w": "self_attn.out_proj.weight",
             "out_b": "self_attn.out_proj.bias", "w1": "linear1.weight", "b1": "linear1.bias", "w2": "linear2.weight",
             "b2": "linear2.bias", "g1": "norm1.weight", "be1": "norm1.bias", "g2": "norm2.weight", "be2": "norm2.bias"}
    for i, lp in enumerate(P["layers"]):
        leaves.update({f"transformer_encoder.layers.{i}.{v}": lp[k] for k, v in names.items()})
    for t in leaves.values():
        t.requires_grad_(True)
    return leaves


@pytest.mark.parametrize("emsize,nhead,precision", [(256, 2, "bf16"), (128, 2, "fp32")])
def test_ragged_forward_and_masked_bar_nll_match_the_oracle(cuda_device, emsize, nhead, precision):
    """A ragged forward plus a masked bar-NLL backward against the fp64 oracle run one dataset at a time at its own
    single_eval_pos: the query-row logits per element, every parameter gradient per tensor, and the logits also against
    the model's own scalar call per dataset.  Rows that are not queries get exactly zero gradient."""
    T, B, n_out = 140, 5, 20
    seps = [0, 140, 33, 70, 129]
    m = _model(cuda_device, emsize, nhead, precision, n_out=n_out)
    with torch.no_grad():      # the reference zero-initialises out_proj / linear2: give them weight so every path matters
        for layer in m.transformer_encoder.layers:
            layer.linear2.weight.normal_(0, 0.05)
            layer.self_attn.out_proj.weight.normal_(0, 0.05)
    m.eval()
    crit = bar_distribution.BarDistribution(BORDERS).to(cuda_device)
    x, y = _data(cuda_device, T, B)
    y = y.clamp(-2.9, 2.9)
    out = m((x, y), single_eval_pos=seps)
    s_min = min(seps)
    assert out.shape == (T - s_min, B, n_out)
    query = m.query_rows(T, seps).to(cuda_device)
    n_query = int(query.sum())
    out.retain_grad()
    losses = crit(out.reshape(-1, n_out), y[s_min:].flatten()).view(T - s_min, B)
    (torch.where(query, losses, 0.).sum() / n_query).backward()
    assert torch.equal(out.grad[~query], torch.zeros_like(out.grad[~query]))
    # the oracle: dataset by dataset at its own separator, one fp64 graph for the summed loss
    P = O.params_from_state_dict(m.state_dict(), 2)
    leaves = _oracle_leaves(P)
    xd, yd = x.double().cpu(), y.double().cpu()
    ref_loss = 0.0
    for b, s in enumerate(seps):
        if s == T:
            continue
        ref = O.transformer_forward_ref(P, xd[:, b:b + 1], yd[:, b:b + 1], s, nhead)
        got = out[s - s_min:, b].detach().cpu()
        EB.check(f"ragged logits b={b} sep={s} {precision}", got, ref[:, 0].detach(),
                 UNIT[precision] * (ref[:, 0].detach().abs() + ref[:, 0].detach().abs().mean()), C_MODEL[precision])
        with torch.no_grad():
            alone = m((x[:, b:b + 1], y[:, b:b + 1]), single_eval_pos=s)[:, 0].cpu()
        EB.check(f"ragged vs scalar call b={b} sep={s} {precision}", got, alone.double(),
                 UNIT[precision] * (alone.double().abs() + alone.double().abs().mean()), C_MODEL[precision])
        ref_loss = ref_loss + O.bar_nll_ref(ref.reshape(-1, n_out), yd[s:, b], BORDERS.double()).sum()
    (ref_loss / n_query).backward()
    named = dict(m.named_parameters())
    for k, t in leaves.items():
        got = named[k].grad.double().cpu()
        scale = t.grad.abs().max().item() + 1e-9
        err = (got - t.grad).abs().max().item()
        assert err <= C_GRAD[precision] * scale, f"{k}: {err} vs scale {scale}"


def test_forward_rejects_bad_vectors(cuda_device):
    m = _model(cuda_device, 128, 2, "bf16")
    x, y = _data(cuda_device, 20, 3)
    with pytest.raises(ValueError, match="holds 2 values"):
        m((x, y), single_eval_pos=[1, 2])
    with pytest.raises(ValueError, match=r"\[0, 20\]"):
        m((x, y), single_eval_pos=[1, 2, 21])
    with pytest.raises(NotImplementedError):
        m((x, y), single_eval_pos=[1, 2, 3], src_mask=TransformerModel.generate_D_q_matrix(20, 19).to(cuda_device))


# ---- train() ----------------------------------------------------------------------------------------------------------
def _train_kwargs(crit, gen, batch_size=16):
    return dict(criterion=crit, encoder_generator=encoders.Linear, emsize=128, nhid=256, nlayers=2, nhead=1, dropout=0.0,
                epochs=2, steps_per_epoch=4, batch_size=batch_size, bptt=30, lr=1e-3, warmup_epochs=0,
                y_encoder_generator=encoders.Linear,
                extra_prior_kwargs_dict={"num_features": 1, "hyperparameters": {"noise": .1, "outputscale": .1, "lengthscale": .1}},
                single_eval_pos_gen=gen, verbose=False)


def _bar(dev):
    torch.manual_seed(0)
    ys = priors.fast_gp.get_batch(200, 30, 1, device=dev)[1]
    return bar_distribution.FullSupportBarDistribution(bar_distribution.get_bucket_limits(50, ys=ys.cpu()))


def test_train_with_per_dataset_sampler(cuda_device):
    crit = _bar(cuda_device)
    torch.manual_seed(0); random.seed(0)
    gen = utils.per_dataset_sampler(utils.get_weighted_single_eval_pos_sampler(30), 16)
    total_loss, pos_losses, model = train_mod.train(priors.fast_gp.DataLoader, **_train_kwargs(crit, gen))
    assert total_loss == total_loss and abs(total_loss) < 1e3
    assert len(pos_losses) == 30


def test_train_constant_vector_is_the_scalar_step(cuda_device):
    """A vector of equal values takes the scalar step: the same loss bit for bit, and the same gradients up to the order
    of the split-K weight-gradient reductions, which differs from one run of the scalar step to the next."""
    crit = _bar(cuda_device)
    torch.manual_seed(0); random.seed(0)
    tr = train_mod.build_trainer(priors.fast_gp.DataLoader, **_train_kwargs(crit, lambda: 12))
    tr.aggregate_k_gradients = 1000         # no optimizer step: both calls see the same weights
    data, targets = next(iter(tr.dl))
    res = []
    for sep in (12, [12] * 16):
        tr.model.zero_grad()
        loss, _ = tr.step(data, targets, sep)
        res.append((loss.detach(), _grads(tr.model)))
    assert torch.equal(res[0][0], res[1][0])
    for n, ref in res[0][1].items():
        assert (res[1][1][n] - ref).abs().max() <= 1e-5 * ref.abs().amax().clamp(min=1e-6), n


def test_trainer_loss_is_the_query_row_mean(cuda_device):
    """The Trainer's loss on a ragged step is the mean of the per-row losses over the query rows of the batch."""
    crit = _bar(cuda_device)
    torch.manual_seed(0); random.seed(0)
    tr = train_mod.build_trainer(priors.fast_gp.DataLoader, **_train_kwargs(crit, lambda: 0, batch_size=4))
    tr.optimizer.param_groups[0]["lr"] = 0.0
    data, targets = next(iter(tr.dl))
    seps = [3, 29, 10, 0]
    loss, losses = tr.step(data, targets, seps)
    query = tr.model.query_rows(30, seps).to(losses.device)
    assert torch.allclose(loss, losses[query].mean(), rtol=1e-5)
    with pytest.raises(ValueError, match="no query row"):
        tr.step(data, targets, [30] * 4)


def test_two_gpu_ragged_step_gradient():
    """Data parallel on 2 GPUs (NCCL; skipped below 2 devices): Trainer.step with one value per dataset of the global
    batch, through the overlapped bucketed all-reduce, gives the single-device gradient of the global batch's masked
    mean, also when one rank's slice has no query row (tests/dp_ragged_worker.py)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29713", os.path.join(root, "tests", "dp_ragged_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "DP_RAGGED_WORKER_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
