"""Input gradients on the H100: the context-attention backward (csrc/attention_bwd_tc.cu, attention_simt.cu) and the
embedding's input gradient (csrc/rowwise.cu) against fp64 restatements, and `forward` / `predict` differentiated in their
inputs against fp64 autograd through the oracle, with the properties a caller of `predict`'s backward relies on: the
parameters' .grad and the context are untouched, and the logits are those of the call without a graph."""
import pytest
import torch

from transformerscandobayesianinference_b200 import _lib as L, _lib_input_grad as LIG, bar_distribution, decoders, encoders
from transformerscandobayesianinference_b200 import transformer
from oracle import error_budget as EB, pfn_oracle as O

pytestmark = pytest.mark.gpu

UNIT = {"bf16": EB.U, "fp32": EB.U32}
# Per-element bound on an input gradient of the whole model: c * u * (|ref| + mean |ref|), u the unit roundoff of the
# activation dtype, as the logits' bound of tests/test_gpu_context_inference.py.  c: at least twice the worst ratio
# measured on an H100 80GB HBM3 at a 700 W power limit: bf16 38.9, fp32 353 (dL/dy of forward; predict 6.2 and 36.9).
C_GRAD = {"bf16": 128.0, "fp32": 1024.0}
# The context backward's fp32-FMA path against the fp64 restatement: its dP = dO . v sums dh fp32 products whose
# cancellation the bound's |dP| does not cover, so the fp32 ratios exceed EB.C_ATT_GRAD (worst 9.10, dK, dh 64; the masked
# backward on the same data reaches the same values)
C_ATT_GRAD_FP32 = 20.0
# the embedding input gradient: fp32 sums over E of U32 E |dout| |W| (the kernel's longest path adds E / 32 + 5 terms)
C_EMBED_IN = EB.C_ROWSUM


def _model(E, H, L_, n_out, precision, F=2, seed=0, **kw):
    torch.manual_seed(seed)
    m = transformer.TransformerModel(encoders.Linear(F, E), n_out, E, H, 2 * E, L_, 0.0, y_encoder=encoders.Linear(1, E),
                                     **kw)
    with torch.no_grad():      # the reference zero-initialises out_proj / linear2: give them weight so every path matters
        for layer in m.transformer_encoder.layers:
            layer.linear2.weight.normal_(0, 0.05)
            layer.self_attn.out_proj.weight.normal_(0, 0.05)
    m.precision = precision
    return m.cuda().eval()


def _bound(ref, precision):
    ref = ref.double()
    return UNIT[precision] * (ref.abs() + ref.abs().mean())


# ---- the context-attention backward alone --------------------------------------------------------------------------
def _ctx_operands(n, m, B, H, dh, dtype, g):
    E = H * dh
    qkv = (torch.randn(m * B, 3 * E, device="cuda", generator=g)).to(dtype)
    kv = (torch.randn(max(n, 1) * B, 2 * E, device="cuda", generator=g)).to(dtype)[:n * B]
    dout = torch.randn(m * B, E, device="cuda", generator=g).to(dtype)
    return qkv, kv, dout


def _ctx_fwd_bwd(qkv, kv, dout, m, n, B, H, dh, use_tc, n_keys=None):
    E = H * dh
    out = torch.empty(m * B, E, device="cuda", dtype=qkv.dtype)
    lse = torch.empty(B * H, m, device="cuda")
    LIG.attention_ctx_grad_fwd(qkv, kv, out, lse, m, n, B, H, dh, n_keys, use_tc=use_tc)
    dqkv = torch.full((m * B, 3 * E), float("nan"), device="cuda", dtype=qkv.dtype)
    delta = torch.empty(B * H, m, device="cuda")
    LIG.attention_ctx_bwd(qkv, kv, out, lse, dout, dqkv, delta, m, n, B, H, dh, n_keys, use_tc=use_tc)
    return out, lse, dqkv


def _concat(qkv, kv, n, m, B, E):
    """The sequence (training rows, query rows) as a masked-attention qkv: the training rows' k | v from the cache (their q
    is never read by a query row's result), then the query rows."""
    full = torch.zeros((n + m) * B, 3 * E, device=qkv.device, dtype=qkv.dtype)
    full[:n * B, E:] = kv
    full[n * B:] = qkv
    return full


KERNEL_PATHS = [(torch.bfloat16, 128, True), (torch.bfloat16, 128, False), (torch.bfloat16, 64, False),
                (torch.float32, 64, False), (torch.float32, 128, False)]
# (n, m, B): every training-row count, query-row count and batch of the grid appears, with the 64-row tile edges
CTX_CASES = [(0, 65, 3), (1, 1, 16), (63, 64, 1), (64, 3000, 1), (65, 65, 16), (1000, 64, 3), (1000, 3000, 1)]


@pytest.mark.parametrize("n,m,B", CTX_CASES)
@pytest.mark.parametrize("dtype,dh,use_tc", KERNEL_PATHS)
def test_context_backward_kernel(n, m, B, dtype, dh, use_tc):
    H = 2
    E = H * dh
    g = torch.Generator(device="cuda").manual_seed(n * 31 + m * 7 + B)
    qkv, kv, dout = _ctx_operands(n, m, B, H, dh, dtype, g)
    out, lse, dqkv = _ctx_fwd_bwd(qkv, kv, dout, m, n, B, H, dh, use_tc)
    tag = f" n={n} m={m} B={B} {dtype} dh={dh} {'tc' if use_tc else 'simt'}"
    # the forward's out is the context forward's bit for bit
    plain = torch.empty_like(out)
    L.attention_ctx_fwd(qkv, kv, plain, m, n, B, H, dh, use_tc=use_tc)
    assert torch.equal(out, plain)
    # fp64 restatement: rows n .. n + m - 1 of the masked attention on the concatenated sequence at sep = n; the training
    # rows get a zero output gradient, so they add nothing to any query row's gradient
    u = EB.U if dtype == torch.bfloat16 else EB.U32
    full = _concat(qkv, kv, n, m, B, E)
    f = EB.attention_fwd(full, n + m, B, H, dh, n, u)
    EB.check(f"ctx out{tag}", out, f["out"][n * B:], f["out_bound"][n * B:], EB.C_ATT_OUT)
    EB.check(f"ctx lse{tag}", lse, f["lse"][:, n:], f["lse_bound"][:, n:], EB.C_ATT_LSE)
    dout_full = torch.zeros((n + m) * B, E, device="cuda", dtype=dtype)
    dout_full[n * B:] = dout
    out_full = torch.zeros_like(dout_full)
    out_full[n * B:] = out
    b = EB.attention_bwd(f, dout_full, out_full)
    rows = {k: v[n * B:] for k, v in b.items()}
    c_grad = EB.C_ATT_GRAD if dtype == torch.bfloat16 else C_ATT_GRAD_FP32
    EB.check_attention_bwd(dqkv, rows, c_grad, tag=f" ctx{tag}")
    # the masked backward on the concatenated sequence: its rows >= n hold the same gradients
    o2 = torch.empty((n + m) * B, E, device="cuda", dtype=dtype)
    l2 = torch.empty(B * H, n + m, device="cuda")
    L.attention_fwd(full, o2, l2, n + m, B, H, dh, n, use_tc=use_tc)
    d2 = torch.empty((n + m) * B, 3 * E, device="cuda", dtype=dtype)
    L.attention_bwd(full, o2, l2, dout_full, d2, torch.empty(B * H, n + m, device="cuda"), n + m, B, H, dh, n,
                    use_tc=use_tc)
    EB.check_attention_bwd(d2[n * B:], rows, c_grad, tag=f" masked{tag}")
    print(f"[ctx bwd{tag}] equal to the masked backward's rows >= n bitwise: {torch.equal(d2[n * B:], dqkv)}")


@pytest.mark.parametrize("dtype,dh,use_tc", KERNEL_PATHS)
def test_ragged_context_backward_is_each_datasets_own_call(dtype, dh, use_tc):
    """Column b of a call with n_keys equals the one-dataset call on its first n_keys[b] cached rows, bit for bit."""
    n, m, H = 130, 70, 2
    sizes = [0, 1, 63, 64, 65, 130]
    B, E = len(sizes), H * dh
    g = torch.Generator(device="cuda").manual_seed(5)
    qkv, kv, dout = _ctx_operands(n, m, B, H, dh, dtype, g)
    n_keys = torch.tensor(sizes, dtype=torch.int32, device="cuda")
    out, lse, dqkv = _ctx_fwd_bwd(qkv, kv, dout, m, n, B, H, dh, use_tc, n_keys)
    for b, nb in enumerate(sizes):
        q1 = qkv.view(m, B, 3 * E)[:, b].contiguous()
        kv1 = kv.view(n, B, 2 * E)[:nb, b].contiguous()
        d1 = dout.view(m, B, E)[:, b].contiguous()
        o1, l1, g1 = _ctx_fwd_bwd(q1, kv1, d1, m, nb, 1, H, dh, use_tc)
        assert torch.equal(out.view(m, B, E)[:, b], o1), b
        assert torch.equal(dqkv.view(m, B, 3 * E)[:, b], g1), b


# ---- the embedding's input gradient ----------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("T,B,F,E,sep", [(10, 4, 1, 128, 4), (7, 3, 5, 96, 0), (9, 2, 18, 512, 9), (33, 5, 64, 40, 2),
                                         (300, 16, 33, 512, 100)])
@pytest.mark.parametrize("ragged", [False, True])
def test_embed_input_grad(dtype, T, B, F, E, sep, ragged):
    g = torch.Generator(device="cuda").manual_seed(T * B + F)
    dout = torch.randn(T * B, E, device="cuda", generator=g).to(dtype)
    Wx, wy = torch.randn(E, F, device="cuda", generator=g), torch.randn(E, device="cuda", generator=g)
    n_keys = torch.randint(0, T + 1, (B,), device="cuda", generator=g, dtype=torch.int32) if ragged else None
    runs = []
    for _ in range(2):
        dx, dy = torch.empty(T * B, F, device="cuda"), torch.empty(T * B, device="cuda")
        LIG.embed_input_bwd(dout, Wx, wy, dx, dy, T, B, F, E, sep, n_keys)
        runs.append((dx, dy))
    assert all(torch.equal(a, b) for a, b in zip(*runs))        # a fixed reduction order
    d, W, w = dout.double(), Wx.double(), wy.double()
    t = torch.arange(T, device="cuda").repeat_interleave(B)
    train = (t < (n_keys.long().repeat(T) if ragged else sep)).double()
    tag = f" T={T} B={B} F={F} E={E} {dtype}{' ragged' if ragged else ''}"
    EB.check(f"embed dx{tag}", dx, d @ W, EB.U32 * E * (d.abs() @ W.abs()), C_EMBED_IN)
    EB.check(f"embed dy{tag}", dy, train * (d @ w), EB.U32 * E * train * (d.abs() @ w.abs()), C_EMBED_IN)


# ---- the model -------------------------------------------------------------------------------------------------------
def _oracle_input_grads(model, x, y, sep, W):
    """fp64 autograd of sum(logits * W) through the oracle at scalar sep: (dL/dx, dL/dy)."""
    P = O.params_from_state_dict(model.state_dict(), len(model.transformer_encoder.layers))
    xr = x.detach().cpu().double().requires_grad_(True)
    yr = y.detach().cpu().double().requires_grad_(True)
    ref = O.transformer_forward_ref(P, xr, yr, sep, model.nhead)
    (ref * W.cpu().double()).sum().backward()
    return xr.grad, yr.grad


def _predict_grad(model, ctx, xq, W=None, loss=None):
    xq = xq.detach().clone().requires_grad_(True)
    out = model.predict(ctx, xq)
    (loss(out) if loss else (out * W).sum()).backward()
    return out, xq.grad


# (n, m, B) of the model tests
MODEL_CASES = [(0, 65, 3), (1, 1, 1), (64, 64, 3), (65, 200, 16), (1000, 300, 1)]


@pytest.mark.parametrize("n,m,B", MODEL_CASES)
@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_predict_and_forward_input_grads_match_oracle(n, m, B, dh, precision):
    H = 2
    model = _model(H * dh, H, 2, 20, precision, seed=n + m + B)
    g = torch.Generator(device="cuda").manual_seed(n * 7 + m)
    x = torch.rand(n + m, B, 2, device="cuda", generator=g)
    y = torch.randn(n + m, B, device="cuda", generator=g)
    W = torch.randn(m, B, 20, device="cuda", generator=g)
    gx_ref, gy_ref = _oracle_input_grads(model, x, y, n, W)
    tag = f" n={n} m={m} B={B} dh={dh} {precision}"
    with torch.no_grad():
        ctx = model.encode_context(x[:n], y[:n])
    _, gq = _predict_grad(model, ctx, x[n:], W)
    EB.check(f"predict dx{tag}", gq.cpu(), gx_ref[n:], _bound(gx_ref[n:], precision), C_GRAD[precision])
    xf, yf = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    (model((xf, yf), single_eval_pos=n) * W).sum().backward()
    EB.check(f"forward dx{tag}", xf.grad.cpu(), gx_ref, _bound(gx_ref, precision), C_GRAD[precision])
    EB.check(f"forward dy{tag}", yf.grad.cpu(), gy_ref, _bound(gy_ref, precision), C_GRAD[precision])
    assert not yf.grad[n:].any()
    print(f"[predict vs forward{tag}] x[n:].grad bitwise equal: {torch.equal(gq, xf.grad[n:])}")


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_forward_input_grads_per_dataset_seps(dh, precision):
    """forward with one single_eval_pos per dataset against the oracle run on each dataset at its own value."""
    H, T = 2, 200
    seps = [0, 1, 63, 64, 130, 199]
    B = len(seps)
    model = _model(H * dh, H, 2, 20, precision, seed=3)
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.rand(T, B, 2, device="cuda", generator=g)
    y = torch.randn(T, B, device="cuda", generator=g)
    s_min = min(seps)
    W = torch.randn(T - s_min, B, 20, device="cuda", generator=g) * transformer.TransformerModel.query_rows(T, seps).cuda()[
        ..., None]
    xf, yf = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    (model((xf, yf), single_eval_pos=seps) * W).sum().backward()
    for b, s in enumerate(seps):
        gx_ref, gy_ref = _oracle_input_grads(model, x[:, b:b + 1], y[:, b:b + 1], s, W[s - s_min:, b:b + 1])
        tag = f" sep={s} dh={dh} {precision}"
        EB.check(f"forward ragged dx{tag}", xf.grad[:, b:b + 1].cpu(), gx_ref, _bound(gx_ref, precision), C_GRAD[precision])
        EB.check(f"forward ragged dy{tag}", yf.grad[:, b:b + 1].cpu(), gy_ref, _bound(gy_ref, precision), C_GRAD[precision])
        assert not yf.grad[s:, b].any()


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_predict_ragged_context_grad_is_each_datasets_own(precision):
    """predict's x_query.grad against a ragged context equals, per dataset, the gradient against its own context."""
    n, m, H, dh = 100, 50, 2, 128
    sizes = [0, 1, 64, 100]
    B = len(sizes)
    model = _model(H * dh, H, 2, 20, precision, seed=9)
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.rand(n + m, B, 2, device="cuda", generator=g)
    y = torch.randn(n + m, B, device="cuda", generator=g)
    W = torch.randn(m, B, 20, device="cuda", generator=g)
    with torch.no_grad():
        ctx = model.encode_context(x[:n], y[:n], sizes)
    _, gq = _predict_grad(model, ctx, x[n:], W)
    for b, nb in enumerate(sizes):
        gx_ref, _ = _oracle_input_grads(model, torch.cat([x[:nb, b:b + 1], x[n:, b:b + 1]]),
                                        torch.cat([y[:nb, b:b + 1], y[n:, b:b + 1]]), nb, W[:, b:b + 1])
        EB.check(f"predict ragged dx n_b={nb} {precision}", gq[:, b:b + 1].cpu(), gx_ref[nb:], _bound(gx_ref[nb:], precision),
                 C_GRAD[precision])


@pytest.mark.parametrize("decoder", [decoders.ScaledDecoder, decoders.FixedScaledDecoder])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_scaled_heads_predict_grad_matches_forward(decoder, precision):
    model = _model(256, 2, 2, 30, precision, decoder=decoder)
    x, y = torch.rand(300, 3, 2, device="cuda"), torch.randn(300, 3, device="cuda")
    W = torch.randn(200, 3, 30, device="cuda")
    with torch.no_grad():
        ctx = model.encode_context(x[:100], y[:100])
    _, gq = _predict_grad(model, ctx, x[100:], W)
    model.zero_grad(set_to_none=True)
    xf = x.clone().requires_grad_(True)
    (model((xf, y), single_eval_pos=100) * W).sum().backward()
    ref = xf.grad[100:].double().cpu()
    EB.check(f"{decoder.__name__} predict dx vs forward {precision}", gq.cpu(), ref, _bound(ref, precision),
             C_GRAD[precision])


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_expected_improvement_gradient(precision):
    """d ei(predict(ctx, x), best_f) / dx, the loss a candidate-point optimiser differentiates, against the oracle."""
    n, m, B, n_out = 200, 64, 2, 50
    model = _model(256, 2, 2, n_out, precision, seed=4)
    crit = bar_distribution.BarDistribution(bar_distribution.get_bucket_limits(n_out, full_range=(-3., 3.))).cuda()
    g = torch.Generator(device="cuda").manual_seed(8)
    x = torch.rand(n + m, B, 2, device="cuda", generator=g)
    y = torch.randn(n + m, B, device="cuda", generator=g)
    with torch.no_grad():
        ctx = model.encode_context(x[:n], y[:n])
    _, gq = _predict_grad(model, ctx, x[n:], loss=lambda out: crit.ei(out, 0.5).sum())
    P = O.params_from_state_dict(model.state_dict(), len(model.transformer_encoder.layers))
    xr = x.detach().cpu().double().requires_grad_(True)
    ref = O.transformer_forward_ref(P, xr, y.cpu().double(), n, model.nhead)
    lo, hi = crit.borders[:-1].cpu().double(), crit.borders[1:].cpu().double()
    contrib = ((hi + torch.maximum(lo, torch.tensor(0.5, dtype=torch.float64))) / 2 - 0.5).clamp(min=0)
    (torch.softmax(ref, -1) @ contrib).sum().backward()
    EB.check(f"ei dx {precision}", gq.cpu(), xr.grad[n:], _bound(xr.grad[n:], precision), C_GRAD[precision])


# ---- properties ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("decoder", [None, decoders.ScaledDecoder, decoders.FixedScaledDecoder])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_predict_backward_leaves_parameters_and_context_alone(decoder, precision, monkeypatch):
    model = _model(256, 2, 3, 20, precision, seed=6, **({"decoder": decoder} if decoder else {}))
    x, y = torch.rand(150, 4, 2, device="cuda"), torch.randn(150, 4, device="cuda")
    with torch.no_grad():
        ctx = model.encode_context(x[:100], y[:100], [100, 3, 64, 0])
    kv0 = ctx.kv.clone()
    for i, p in enumerate(model.parameters()):      # some .grad set, some None: both must survive
        p.grad = torch.full_like(p, float(i)) if i % 2 else None
    grads0 = [None if p.grad is None else p.grad.clone() for p in model.parameters()]
    with torch.no_grad():
        plain = model.predict(ctx, x[100:])
    names = []
    real_call = LIG._call
    monkeypatch.setattr(LIG, "_call", lambda name, *a, **k: (names.append(name), real_call(name, *a, **k))[1])
    xq = x[100:].clone().requires_grad_(True)
    out = model.predict(ctx, xq)
    assert torch.equal(out, plain)
    out.sum().backward()
    assert xq.grad is not None and torch.isfinite(xq.grad).all()
    assert torch.equal(ctx.kv, kv0)
    for p, g0 in zip(model.parameters(), grads0):
        assert (p.grad is None) == (g0 is None) and (g0 is None or torch.equal(p.grad, g0))
    n_layers = len(model.transformer_encoder.layers)
    assert sum(nm.startswith("pfn_attention_ctx_bwd") for nm in names) == n_layers
    assert sum(nm.startswith("pfn_attention_ctx_grad_fwd") for nm in names) == n_layers


def test_forward_without_input_grad_launches_as_before():
    """With inputs that do not require grad, the training step's backward makes the same library calls as before: no
    embedding input-gradient launch."""
    model = _model(256, 2, 2, 20, "bf16").train()
    x, y = torch.rand(100, 3, 2, device="cuda"), torch.randn(100, 3, device="cuda")
    L.reset_launch_count()
    model((x, y), single_eval_pos=40).sum().backward()
    base = L.launch_count()
    L.reset_launch_count()
    model((x.clone().requires_grad_(True), y), single_eval_pos=40).sum().backward()
    assert L.launch_count() == base + 1


def test_conv_encoder_still_rejects_input_grad():
    torch.manual_seed(1)
    S, E = 12, 256
    model = transformer.TransformerModel(encoders.Conv(S * S, E), 10, E, 2, 2 * E, 2, 0.0,
                                         y_encoder=encoders.Linear(1, E)).cuda().eval()
    x, y = torch.rand(60, 2, S * S, device="cuda"), torch.randn(60, 2, device="cuda")
    with torch.no_grad():
        ctx = model.encode_context(x[:40], y[:40])
    with pytest.raises(ValueError, match="no gradient for its input"):
        model.predict(ctx, x[40:].clone().requires_grad_(True))
