"""Inference against a cached training set on the H100: `TransformerModel.encode_context` / `predict` against `forward`
on the concatenated sequence and the fp64 oracle, the context-attention kernels (csrc/attention_tc.cu, attention_simt.cu)
against an fp64 restatement, and the properties a caller relies on: query rows are independent of each other, and a
context is reusable and never written."""
import os

import pytest
import torch

from transformerscandobayesianinference_b200 import _lib as L, decoders, encoders, positional_encodings, transformer
from oracle import error_budget as EB, pfn_oracle as O
from oracle.make_golden import build_case_weights, case_inputs

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")

# Per-element bound on logits of the whole model: c * u * (|ref| + mean |ref|), u the unit roundoff of the activation
# dtype.  `predict` and `forward` are held to the same bound against the fp64 oracle (worst on an H100: bf16 11.1, fp32
# 93.6, forward and predict alike).
C_MODEL = {"bf16": 16.0, "fp32": 512.0}
UNIT = {"bf16": EB.U, "fp32": EB.U32}


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


def _check_against_forward_and_oracle(tag, model, x_tr, y_tr, x_q, precision, oracle=True):
    n = x_tr.shape[0]
    with torch.no_grad():
        ctx = model.encode_context(x_tr, y_tr)
        got = model.predict(ctx, x_q)
        y_any = torch.cat([y_tr, torch.randn(x_q.shape[0], x_q.shape[1], device=x_q.device)], 0)
        fwd = model((torch.cat([x_tr, x_q], 0), y_any), single_eval_pos=n)
    assert got.shape == fwd.shape == (x_q.shape[0], x_q.shape[1], fwd.shape[-1])
    print(f"[{tag}] predict == forward bitwise: {torch.equal(got, fwd)}")
    if oracle:
        P = O.params_from_state_dict(model.state_dict(), len(model.transformer_encoder.layers))
        ref = O.transformer_forward_ref(P, torch.cat([x_tr, x_q], 0).cpu().double(), y_any.cpu().double(), n, model.nhead)
    else:          # heads and encoders the oracle does not restate: forward is the reference
        ref = fwd.double().cpu()
    bound = _bound(ref, precision)
    EB.check(f"{tag} predict", got.cpu(), ref, bound, C_MODEL[precision])
    if oracle:
        EB.check(f"{tag} forward", fwd.cpu(), ref, bound, C_MODEL[precision])


# (n, m, B): every training-row count, query-row count and batch of the grid appears, with the ragged 64-row tile edges
CASES = [(0, 65, 3), (1, 1, 1), (17, 63, 16), (64, 64, 3), (64, 65, 1), (1000, 65, 16), (17, 3000, 3), (1000, 3000, 1)]


@pytest.mark.parametrize("n,m,B", CASES)
@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_predict_matches_forward_and_oracle(n, m, B, dh, precision):
    H = 2
    model = _model(H * dh, H, 2, 20, precision, seed=n + m + B)
    g = torch.Generator(device="cuda").manual_seed(n * 7 + m)
    x = torch.rand(n + m, B, 2, device="cuda", generator=g)
    y = torch.randn(n + m, B, device="cuda", generator=g)
    _check_against_forward_and_oracle(f"n={n} m={m} B={B} dh={dh} {precision}", model, x[:n], y[:n], x[n:], precision)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_checkpoint_shaped_model(precision):
    """The GP-regression model shape (emsize 512, 4 heads, 6 layers) of tests/golden/model_cfg2_b4.pt, split at its sep."""
    case = torch.load(os.path.join(GOLD, "model_cfg2_b4.pt"))["case"]
    ctor = lambda enc, yenc: transformer.TransformerModel(enc, case["n_out"], case["E"], case["H"], case["nhid"], case["L"],
                                                          0.0, y_encoder=yenc)
    model = build_case_weights(ctor, case).cuda().eval()
    model.precision = precision
    x, y = case_inputs(case)
    x, y, n = x.cuda(), y.cuda(), case["sep"]
    _check_against_forward_and_oracle(f"cfg2_b4 {precision}", model, x[:n], y[:n], x[n:], precision)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_scaled_decoder_head(precision):
    model = _model(256, 2, 2, 30, precision, decoder=decoders.ScaledDecoder)
    x, y = torch.rand(300, 3, 2, device="cuda"), torch.randn(300, 3, device="cuda")
    _check_against_forward_and_oracle(f"ScaledDecoder {precision}", model, x[:100], y[:100], x[100:], precision,
                                      oracle=False)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_conv_encoder_model(precision):
    torch.manual_seed(1)
    S, E = 12, 256
    enc = encoders.Conv(S * S, E)
    enc.precision = precision
    model = transformer.TransformerModel(enc, 10, E, 2, 2 * E, 2, 0.0, y_encoder=encoders.Linear(1, E))
    with torch.no_grad():
        for layer in model.transformer_encoder.layers:
            layer.linear2.weight.normal_(0, 0.05)
            layer.self_attn.out_proj.weight.normal_(0, 0.05)
    model.precision = precision
    model = model.cuda().eval()
    x, y = torch.rand(90, 2, S * S, device="cuda"), torch.randn(90, 2, device="cuda")
    _check_against_forward_and_oracle(f"Conv {precision}", model, x[:40], y[:40], x[40:], precision, oracle=False)


# ---- the context-attention kernel alone --------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 200])
@pytest.mark.parametrize("m", [1, 64, 65, 200])
@pytest.mark.parametrize("dtype,dh,use_tc", [(torch.bfloat16, 128, True), (torch.bfloat16, 128, False),
                                             (torch.bfloat16, 64, False), (torch.float32, 64, False),
                                             (torch.float32, 128, False)])
def test_context_attention_kernel(n, m, dtype, dh, use_tc):
    """Row n + i of the masked attention on (training rows, query rows) with sep = n is query row i's context attention:
    error_budget.attention_fwd on the concatenated rows gives the exact output and its bound."""
    B, H = 3, 2
    E = H * dh
    g = torch.Generator(device="cuda").manual_seed(n * 1000 + m + dh)
    full = (torch.randn((n + m) * B, 3 * E, device="cuda", generator=g) * 1.5).to(dtype)
    kv = full[:n * B, E:].contiguous()
    qkv = full[n * B:].contiguous()
    out = torch.full((m * B, E), float("nan"), device="cuda", dtype=dtype)
    L.attention_ctx_fwd(qkv, kv, out, m, n, B, H, dh, use_tc=use_tc)
    f = EB.attention_fwd(full, n + m, B, H, dh, n, EB.U if dtype == torch.bfloat16 else EB.U32)
    EB.check(f"ctx attention n={n} m={m} dh={dh} {dtype} tc={use_tc}", out, f["out"][n * B:], f["out_bound"][n * B:],
             EB.C_ATT_OUT)


def test_context_attention_kernel_rising_max():
    """Key blocks whose running max rises slowly, so that a skipped rescale of O would show."""
    B, H, dh, n, m = 2, 2, 128, 320, 130
    E = H * dh
    full = EB.rising_max_qkv(n + m, B, H, dh, generator=torch.Generator().manual_seed(3), device="cuda")
    out = torch.empty(m * B, E, device="cuda", dtype=torch.bfloat16)
    L.attention_ctx_fwd(full[n * B:].contiguous(), full[:n * B, E:].contiguous(), out, m, n, B, H, dh)
    f = EB.attention_fwd(full, n + m, B, H, dh, n, EB.U)
    EB.check("ctx attention rising max", out, f["out"][n * B:], f["out_bound"][n * B:], EB.C_ATT_OUT)


def test_context_attention_counts_one_launch():
    qkv = torch.randn(64 * 2, 3 * 256, device="cuda", dtype=torch.bfloat16)
    kv = torch.randn(10 * 2, 2 * 256, device="cuda", dtype=torch.bfloat16)
    out = torch.empty(64 * 2, 256, device="cuda", dtype=torch.bfloat16)
    L.reset_launch_count()
    L.attention_ctx_fwd(qkv, kv, out, 64, 10, 2, 2, 128)
    assert L.launch_count() == 1


# ---- properties --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,dh", [("bf16", 128), ("bf16", 64), ("fp32", 128)])
def test_query_rows_are_independent(precision, dh):
    """Every kernel of the query path computes a row from that row alone, in an order that does not depend on the other
    rows: the forward GEMMs run without split-K (engine._linear_fwd: k_splits 1), the attention, LayerNorm and embedding
    kernels are row-wise.  So predicting the queries in chunks gives the very same bits as one call."""
    model = _model(2 * dh, 2, 3, 40, precision, seed=5)
    x, y = torch.rand(500, 4, 2, device="cuda"), torch.randn(500, 4, device="cuda")
    with torch.no_grad():
        ctx = model.encode_context(x[:150], y[:150])
        whole = model.predict(ctx, x[150:])
        parts = [model.predict(ctx, x[a:b]) for a, b in ((150, 151), (151, 214), (214, 278), (278, 500))]
    assert torch.equal(torch.cat(parts, 0), whole)


def test_context_is_reusable_and_unchanged():
    model = _model(256, 2, 2, 20, "bf16", seed=6)
    x, y = torch.rand(300, 3, 2, device="cuda"), torch.randn(300, 3, device="cuda")
    with torch.no_grad():
        ctx = model.encode_context(x[:100], y[:100])
        before = ctx.kv.clone()
        a = model.predict(ctx, x[100:])
        other = model.predict(ctx, x[150:170])
        b = model.predict(ctx, x[100:])
    assert torch.equal(a, b) and torch.equal(other, a[50:70])
    assert torch.equal(ctx.kv, before)
    assert ctx.kv.dtype == torch.bfloat16 and ctx.kv.shape == (2, 100 * 3, 2 * 256)
    assert (ctx.n, ctx.B, ctx.E, ctx.nhead, ctx.nlayers, ctx.precision) == (100, 3, 256, 2, 2, "bf16")


def test_predict_runs_without_autograd():
    model = _model(128, 2, 2, 10, "fp32", seed=7)
    x, y = torch.rand(40, 2, 2, device="cuda"), torch.randn(40, 2, device="cuda")
    ctx = model.encode_context(x[:20], y[:20])
    out = model.predict(ctx, x[20:])
    assert not out.requires_grad and not ctx.kv.requires_grad


# ---- configuration errors ----------------------------------------------------------------------------------------
def test_rejected_configurations_raise_before_any_launch():
    x, y = torch.rand(30, 2, 2, device="cuda"), torch.randn(30, 2, device="cuda")
    bad = [
        _model(128, 2, 2, 10, "bf16", input_normalization=True),
        _model(128, 2, 2, 10, "bf16", pos_encoder=positional_encodings.PositionalEncoding(128, 100)),
        _model(128, 2, 2, 10, "bf16", pos_encoder=positional_encodings.LearnedPositionalEncoding(128, 100)),
    ]
    dropout = _model(128, 2, 2, 10, "bf16")
    dropout.dropout = 0.1
    bad.append(dropout.train())
    good = _model(128, 2, 2, 10, "bf16")
    ctx = good.encode_context(x[:10], y[:10])
    for m in bad:
        L.reset_launch_count()
        with pytest.raises(ValueError):
            m.encode_context(x[:10], y[:10])
        with pytest.raises(ValueError):
            m.predict(ctx, x[10:])
        assert L.launch_count() == 0


def test_context_mismatches_raise():
    x, y = torch.rand(30, 2, 2, device="cuda"), torch.randn(30, 2, device="cuda")
    model = _model(128, 2, 2, 10, "bf16")
    ctx = model.encode_context(x[:10], y[:10])
    others = {"E": _model(256, 2, 2, 10, "bf16"), "nhead": _model(128, 4, 2, 10, "bf16"),
              "nlayers": _model(128, 2, 3, 10, "bf16"), "precision": _model(128, 2, 2, 10, "fp32")}
    for name, m in others.items():
        L.reset_launch_count()
        with pytest.raises(ValueError, match=name):
            m.predict(ctx, x[10:])
        assert L.launch_count() == 0
    with pytest.raises(ValueError, match="B"):
        model.predict(ctx, torch.rand(5, 3, 2, device="cuda"))
    with pytest.raises(ValueError, match="device"):
        model.predict(ctx, x[10:].cpu())
