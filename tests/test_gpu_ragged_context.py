"""Training sets of different sizes in one batch on the H100: `encode_context(x_train, y_train, n_train)` / `predict`
against one-dataset calls, `forward` and the fp64 oracle, the ragged attention kernels (csrc/attention_tc.cu,
attention_simt.cu) against an fp64 restatement per dataset, and the properties a caller relies on: padding never reaches
an output, and sizes that are all n change nothing."""
import pytest
import torch

from transformerscandobayesianinference_b200 import _lib as L, _lib_ragged as LR, encoders, transformer
from oracle import error_budget as EB, pfn_oracle as O

pytestmark = pytest.mark.gpu

# the per-element bound of tests/test_gpu_context_inference.py: c * u * (|ref| + mean |ref|)
C_MODEL = {"bf16": 16.0, "fp32": 512.0}
UNIT = {"bf16": EB.U, "fp32": EB.U32}
N = 100
SIZES = [0, 1, 63, 64, 65, N]          # both sides of the 64-key block edge, an empty and a full training set


def _model(E, H, L_, n_out, precision, F=2, seed=0):
    torch.manual_seed(seed)
    m = transformer.TransformerModel(encoders.Linear(F, E), n_out, E, H, 2 * E, L_, 0.0, y_encoder=encoders.Linear(1, E))
    with torch.no_grad():      # the reference zero-initialises out_proj / linear2: give them weight so every path matters
        for layer in m.transformer_encoder.layers:
            layer.linear2.weight.normal_(0, 0.05)
            layer.self_attn.out_proj.weight.normal_(0, 0.05)
    m.precision = precision
    return m.cuda().eval()


def _bound(ref, precision):
    ref = ref.double()
    return UNIT[precision] * (ref.abs() + ref.abs().mean())


def _data(B, m, seed, F=2):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x_tr, y_tr = torch.rand(N, B, F, device="cuda", generator=g), torch.randn(N, B, device="cuda", generator=g)
    x_q, y_any = torch.rand(m, B, F, device="cuda", generator=g), torch.randn(m, B, device="cuda", generator=g)
    return x_tr, y_tr, x_q, y_any


# ---- the model ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,dh", [("bf16", 128), ("bf16", 64), ("fp32", 64), ("fp32", 128)])
def test_each_dataset_matches_its_own_calls_forward_and_oracle(precision, dh):
    """Column b of one ragged call against dataset b on its own:
    - encode_context + predict on its n_b rows (B = 1): the same kernels compute every row from the same operands in the
      same order (the GEMMs have no split-K, LayerNorm and embedding are row-wise, the attention walks the same 64-key
      blocks), so the bits are equal;
    - forward at single_eval_pos = n_b and the fp64 oracle: the bound of the uniform context tests.  forward runs the
      masked attention on the concatenated rows instead of the context attention on the cache; equal bits are usual
      there too but not promised, as for the uniform context."""
    H, m = 2, 70
    model = _model(H * dh, H, 2, 20, precision, seed=dh)
    x_tr, y_tr, x_q, y_any = _data(len(SIZES), m, dh)
    P = O.params_from_state_dict(model.state_dict(), 2)
    with torch.no_grad():
        ctx = model.encode_context(x_tr, y_tr, SIZES)
        got = model.predict(ctx, x_q)
        for b, n_b in enumerate(SIZES):
            xs, ys, xq = x_tr[:n_b, b:b + 1], y_tr[:n_b, b:b + 1], x_q[:, b:b + 1]
            alone = model.predict(model.encode_context(xs, ys), xq)[:, 0]
            assert torch.equal(got[:, b], alone), (precision, dh, n_b)
            fwd = model((torch.cat([xs, xq], 0), torch.cat([ys, y_any[:, b:b + 1]], 0)), single_eval_pos=n_b)[:, 0]
            ref = O.transformer_forward_ref(P, torch.cat([xs, xq], 0).cpu().double(),
                                            torch.cat([ys, y_any[:, b:b + 1]], 0).cpu().double(), n_b, model.nhead)[:, 0]
            tag = f"n_b={n_b} dh={dh} {precision}"
            print(f"[{tag}] ragged predict == forward bitwise: {torch.equal(got[:, b], fwd)}")
            bound = _bound(ref, precision)
            EB.check(f"{tag} ragged predict", got[:, b].cpu(), ref, bound, C_MODEL[precision])
            EB.check(f"{tag} ragged vs forward", got[:, b].cpu(), fwd.double().cpu(), _bound(fwd, precision).cpu(),
                     C_MODEL[precision])


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_padding_never_reaches_an_output(precision):
    model = _model(256, 2, 3, 20, precision, seed=3)
    x_tr, y_tr, x_q, _ = _data(len(SIZES), 40, 11)
    sizes = torch.tensor(SIZES)
    pad = torch.arange(N).unsqueeze(1) >= sizes
    with torch.no_grad():
        clean = model.predict(model.encode_context(x_tr, y_tr, SIZES), x_q)
        for fill in (float("nan"), float("inf"), -float("inf"), 1e30):
            xd, yd = x_tr.clone(), y_tr.clone()
            xd[pad.cuda()] = fill
            yd[pad.cuda()] = fill
            got = model.predict(model.encode_context(xd, yd, sizes.cuda()), x_q)
            assert torch.equal(got, clean), fill
    assert torch.isfinite(clean).all()


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_sizes_all_n_is_the_uniform_call(precision):
    """n_train=None and n_train = [n] * B run today's kernels: the same launches and the same bits."""
    model = _model(256, 2, 2, 20, precision, seed=4)
    x_tr, y_tr, x_q, _ = _data(3, 50, 5)
    outs, launches = [], []
    with torch.no_grad():
        for kw in ({}, {"n_train": None}, {"n_train": [N] * 3}, {"n_train": torch.full((3,), N, device="cuda")}):
            L.reset_launch_count()
            ctx = model.encode_context(x_tr, y_tr, **kw)
            outs.append(model.predict(ctx, x_q))
            launches.append(L.launch_count())
            assert ctx.n_train is None
    assert all(torch.equal(o, outs[0]) for o in outs) and len(set(launches)) == 1


def test_ragged_call_launches_what_the_uniform_call_launches():
    """The sizes reach only the attention: one ragged attention launch per layer, every other kernel as before."""
    model = _model(256, 2, 3, 20, "bf16", seed=6)
    x_tr, y_tr, x_q, _ = _data(len(SIZES), 30, 7)
    with torch.no_grad():
        counts = []
        for sizes in (None, SIZES):
            L.reset_launch_count()
            ctx = model.encode_context(x_tr, y_tr, sizes)
            model.predict(ctx, x_q)
            counts.append(L.launch_count())
    assert counts[0] == counts[1]


# ---- the ragged attention kernels alone --------------------------------------------------------------------------
KERNEL_PATHS = [(torch.bfloat16, 128, True), (torch.bfloat16, 128, False), (torch.bfloat16, 64, False),
                (torch.float32, 64, False), (torch.float32, 128, False)]


@pytest.mark.parametrize("dtype,dh,use_tc", KERNEL_PATHS)
def test_ragged_attention_kernel(dtype, dh, use_tc):
    """Dataset b of the ragged masked attention is the masked attention of its own rows at sep = n_b."""
    T, H = 130, 2
    sizes = [0, 1, 63, 64, 65, 128, 130]
    B, E = len(sizes), H * dh
    g = torch.Generator(device="cuda").manual_seed(dh)
    qkv = (torch.randn(T * B, 3 * E, device="cuda", generator=g) * 1.5).to(dtype)
    out = torch.full((T * B, E), float("nan"), device="cuda", dtype=dtype)
    LR.attention_ragged_fwd(qkv, out, T, B, H, dh, torch.tensor(sizes, dtype=torch.int32, device="cuda"), use_tc=use_tc)
    for b, n_b in enumerate(sizes):
        f = EB.attention_fwd(qkv.view(T, B, 3 * E)[:, b].contiguous(), T, 1, H, dh, n_b,
                             EB.U if dtype == torch.bfloat16 else EB.U32)
        EB.check(f"ragged attention n_b={n_b} dh={dh} {dtype} tc={use_tc}", out.view(T, B, E)[:, b], f["out"],
                 f["out_bound"], EB.C_ATT_OUT)


@pytest.mark.parametrize("dtype,dh,use_tc", KERNEL_PATHS)
def test_ragged_context_attention_kernel(dtype, dh, use_tc):
    """Query row i of dataset b attends to the first n_b cached keys and itself: row n_b + i of the masked attention on
    (those cached rows, the query rows) at sep = n_b."""
    n, m, H = 130, 70, 2
    sizes = [0, 1, 63, 64, 65, 130]
    B, E = len(sizes), H * dh
    g = torch.Generator(device="cuda").manual_seed(dh + 1)
    kv = (torch.randn(n * B, 2 * E, device="cuda", generator=g) * 1.5).to(dtype)
    qkv = (torch.randn(m * B, 3 * E, device="cuda", generator=g) * 1.5).to(dtype)
    out = torch.full((m * B, E), float("nan"), device="cuda", dtype=dtype)
    LR.attention_ctx_ragged_fwd(qkv, kv, out, m, n, B, H, dh, torch.tensor(sizes, dtype=torch.int32, device="cuda"),
                                use_tc=use_tc)
    for b, n_b in enumerate(sizes):
        train = torch.cat([torch.zeros(n_b, E, device="cuda", dtype=dtype), kv.view(n, B, 2 * E)[:n_b, b]], 1)
        full = torch.cat([train, qkv.view(m, B, 3 * E)[:, b]], 0)
        f = EB.attention_fwd(full, n_b + m, 1, H, dh, n_b, EB.U if dtype == torch.bfloat16 else EB.U32)
        EB.check(f"ragged ctx attention n_b={n_b} dh={dh} {dtype} tc={use_tc}", out.view(m, B, E)[:, b],
                 f["out"][n_b:], f["out_bound"][n_b:], EB.C_ATT_OUT)


@pytest.mark.parametrize("dtype,dh,use_tc", KERNEL_PATHS)
def test_full_sizes_give_the_uniform_kernels_bits(dtype, dh, use_tc):
    T, m, B, H = 130, 70, 3, 2
    E = H * dh
    g = torch.Generator(device="cuda").manual_seed(dh + 2)
    qkv = torch.randn(T * B, 3 * E, device="cuda", generator=g).to(dtype)
    kv = torch.randn(T * B, 2 * E, device="cuda", generator=g).to(dtype)
    q = torch.randn(m * B, 3 * E, device="cuda", generator=g).to(dtype)
    full = torch.full((B,), T, dtype=torch.int32, device="cuda")
    a, r = torch.empty(T * B, E, device="cuda", dtype=dtype), torch.empty(T * B, E, device="cuda", dtype=dtype)
    L.attention_fwd(qkv, a, torch.empty(B * H, T, device="cuda"), T, B, H, dh, T, use_tc=use_tc)
    LR.attention_ragged_fwd(qkv, r, T, B, H, dh, full, use_tc=use_tc)
    assert torch.equal(a, r)
    a, r = torch.empty(m * B, E, device="cuda", dtype=dtype), torch.empty(m * B, E, device="cuda", dtype=dtype)
    L.attention_ctx_fwd(qkv=q, kv=kv, out=a, m=m, n=T, B=B, H=H, dh=dh, use_tc=use_tc)
    LR.attention_ctx_ragged_fwd(q, kv, r, m, T, B, H, dh, full, use_tc=use_tc)
    assert torch.equal(a, r)


def test_ragged_attention_counts_one_launch():
    qkv = torch.randn(64 * 2, 3 * 256, device="cuda", dtype=torch.bfloat16)
    kv = torch.randn(10 * 2, 2 * 256, device="cuda", dtype=torch.bfloat16)
    out = torch.empty(64 * 2, 256, device="cuda", dtype=torch.bfloat16)
    sizes = torch.tensor([3, 10], dtype=torch.int32, device="cuda")
    L.reset_launch_count()
    LR.attention_ctx_ragged_fwd(qkv, kv, out, 64, 10, 2, 2, 128, sizes)
    assert L.launch_count() == 1
    LR.attention_ragged_fwd(qkv, out, 64, 2, 2, 128, sizes)
    assert L.launch_count() == 2


def test_invalid_sizes_raise_before_any_launch():
    model = _model(128, 2, 2, 10, "bf16")
    x, y = torch.rand(10, 3, 2, device="cuda"), torch.randn(10, 3, device="cuda")
    for bad in ([1, 2], [1, 2, 11], [-1, 2, 3], torch.tensor([1.0, 2.0, 3.0], device="cuda"),
                torch.tensor([1, 2, 30], device="cuda")):
        L.reset_launch_count()
        with pytest.raises(ValueError):
            model.encode_context(x, y, bad)
        assert L.launch_count() == 0
