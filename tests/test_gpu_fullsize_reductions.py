"""Every reduction over the token axis of one training step at the benchmark's own shapes and batch (bench.CONFIGS),
element by element against fp64: the weight gradients (split-K wgmma GEMMs whose contraction is the step's 512 000 or
262 144 tokens), the bias and LayerNorm gamma / beta gradients, the fused in-projection bias, the embedding gradients,
and one FusedClipAdam step on them.  The batch sets both the contraction length and the launch path of these kernels
(k_splits, the grouped colsum, the count of atomics), which the small-batch stage test (test_gpu_engine_stages.py)
never reaches.

test_fullsize_step_reductions: oracle/engine_stages.ReductionCheck checks each reduction right after its call, from the
call's own operands, and asserts the call plan and every wgrad's k_splits as the step runs; it keeps no activation, so
the step's memory is one benchmark step plus BLOCK tokens of fp64 at a time.  The per-stage worst ratios, the call plan and the k_splits of each
case are printed to the log.  At 512 000 tokens that bound (2^-24 K |A||B| times C_ACC_WGRAD) is wider than the share
of one 64-token k-block, so test_wgrad_splitk_partition_is_exact holds the split-K partition itself to exact integer
sums of random operands at the same shapes and split counts."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import bench
from transformerscandobayesianinference_b200 import _lib as L, bar_distribution, encoders, engine, optim, priors, transformer
from oracle import engine_stages as ES, error_budget as EB

# tokens per fp64 block: the in-projection wgrad holds 65536 x (1536 + 512) operand values in fp64 and their magnitudes,
# about 2.1 GB, the largest of any check
BLOCK = 1 << 16

# cfg2 at p = 0 is the benchmarked path (fused in-projection bias, delta from the out-projection dgrad, GELU' from the
# forward); cfg4 at p = 0.2 the unfused bias (colsum over dqkv) and the dropout sites; cfg3 the 18-feature embedding and
# the single-row BCE decoder W2
CASES = [("cfg2", 0.0), ("cfg4", 0.2), ("cfg3", 0.0)]


def _batch(name, cfg, dev):
    """One batch from the benchmark's prior at the benchmark's batch, and its criterion."""
    torch.manual_seed(41)
    mods = {"priors": priors, "bar_distribution": bar_distribution, "encoders": encoders}
    _, crit, _, kw = bench.trainer_args(name, cfg, cfg["batch"], mods, str(dev), 1)
    pk = {k: v for k, v in kw["extra_prior_kwargs_dict"].items() if k != "num_features"}
    x, y, target = getattr(priors, cfg["prior"]).get_batch(cfg["batch"], cfg["T"], cfg["F"], **pk)
    return x, y, target, crit


def _model(cfg, p, dev):
    torch.manual_seed(42)
    m = transformer.TransformerModel(encoders.Linear(cfg["F"], cfg["E"]), cfg["n_out"], cfg["E"], cfg["H"], cfg["nhid"],
                                     cfg["L"], p, y_encoder=encoders.Linear(1, cfg["E"])).to(dev)
    bench.randomise_zero_init(m)          # out_proj and linear2 carry weight, so every gradient path carries signal
    m.precision = "bf16"
    return m.train()


def _adam_checked(m, chk):
    """One FusedClipAdam step on the step's gradients against EB.adam_step, with the clip engaged (max_grad_norm half
    the gradient norm) and the norm's depth from the chunk count the optimizer launched with."""
    params = [p for p in m.parameters() if p.grad is not None]
    before = [(p.detach().clone(), p.grad.clone()) for p in params]
    norm_sq = sum((g.double() ** 2).sum() for _, g in before).item()
    max_norm, lr = 0.5 * math.sqrt(norm_sq), 1e-4
    opt = optim.FusedClipAdam(params, lr=lr, max_grad_norm=max_norm)
    opt.step()
    torch.cuda.synchronize()
    n_chunks = opt._tables[0][3]
    chunk = L.adam_chunk_elems()
    assert n_chunks == sum((p.numel() + chunk - 1) // chunk for p in params)
    depth = EB.adam_norm_depth(n_chunks)
    got = opt.last_grad_norm_sq.double()
    chk.chk("adam norm_sq", got, torch.full_like(got, norm_sq), torch.full_like(got, EB.U32 * depth * norm_sq), EB.C_ADAM)
    for p, (p0, g) in zip(params, before):
        zero = torch.zeros_like(p0)
        ex = EB.adam_step(p0, g, zero, zero, 1, lr, 0.9, 0.999, 1e-8, 0.0, norm_sq, max_norm, depth)
        st = opt.state[p]
        for key, t in (("p", p.detach()), ("m", st["exp_avg"]), ("v", st["exp_avg_sq"])):
            chk.chk("adam " + key, t, ex[key], ex[key + "_bound"], EB.C_ADAM)


@pytest.mark.parametrize("name,p", CASES)
def test_fullsize_step_reductions(cuda_device, capsys, name, p):
    dev = cuda_device
    cfg = bench.CONFIGS[name]
    x, y, target, crit = _batch(name, cfg, dev)
    m = _model(cfg, p, dev)
    sep, n_out = cfg["sep"], cfg["n_out"]
    # the benchmark's path at these shapes: a path that quietly changes at full size fails the plan
    paths = {"u_is_grad": True, "rowdot": True, "fused_bias": p == 0}
    tag = f"{name} B={cfg['batch']} p={p}"
    chk = ES.ReductionCheck(L, n_layers=cfg["L"], drop=p > 0, paths=paths, head=cfg["head"], num_sms=L.num_sms(),
                            splits=engine._wgrad_splits, block=BLOCK, tag=tag + ": ").install()
    try:
        logits = m((x, y), single_eval_pos=sep)
        t = target[sep:]
        if cfg["head"] == "bar":
            loss = crit(logits.reshape(-1, n_out), t.flatten()).mean()
        else:
            loss = crit(logits.flatten(), t.flatten()).mean()
        loss.backward()
    finally:
        chk.remove()
    torch.cuda.synchronize()
    del logits, loss
    layers = [dict(zip(ES.LAYER_PARAM_NAMES, [t.detach() for t in engine.layer_params(l)])) for l in m.transformer_encoder.layers]
    grads = [dict(zip(ES.LAYER_PARAM_NAMES, [t.grad for t in engine.layer_params(l)])) for l in m.transformer_encoder.layers]
    chk.finish(layers, grads)
    _adam_checked(m, chk)
    pf, pb = ES.layer_plan(p > 0, paths["u_is_grad"], paths["rowdot"], paths["fused_bias"])
    with capsys.disabled():
        print(f"\n[call-plan] {tag}: {len(chk.sigs)} calls as planned; per layer forward {pf}; backward {pb}")
        chk.report(tag)
    n_wgrad = 4 * cfg["L"] + 2
    assert sum(s == "gemm/none/acc" for s in chk.sigs) == n_wgrad
    if L.num_sms() == 132:
        # H100 SXM: the out-projection launches 16 splits and the decoder's W2 33, 63 to 1 600 k-blocks of 64 tokens each
        assert chk.k_splits["dw_out"] == {16} and chk.k_splits["dec dW2"] == {33}


def _wgrad_shapes():
    """(tokens, rows, cols) of every wgrad launch of the benchmark's configurations: the layers' in_w, out_w, w1 and w2
    over all tokens, the decoder's W0 and W2 over the query tokens."""
    shapes = set()
    for c in bench.CONFIGS.values():
        E, nhid, n, nq = c["E"], c["nhid"], c["T"] * c["batch"], (c["T"] - c["sep"]) * c["batch"]
        shapes |= {(n, r, k) for r, k in ((3 * E, E), (E, E), (nhid, E), (E, nhid))}
        shapes |= {(nq, nhid, E), (nq, c["n_out"], nhid)}
    return sorted(shapes)


@pytest.mark.parametrize("K,M,N", _wgrad_shapes())
def test_wgrad_splitk_partition_is_exact(cuda_device, K, M, N):
    """engine._linear_wgrad at the step's shapes and split counts, on operands drawn independently from {1, 2}: every
    partial sum is an integer below 2^24, so fp32 adds them exactly in any order and the result must equal the exact sum
    bit for bit.  Each 64-token k-block contributes its own random amount to each element, and the exact rows and
    128-column blocks are all distinct, so a block lost, counted twice or read from another split's range, a lost
    reduce-add, and a tile stored at another (m0, n0) change the result.  dY is a view of a buffer padded to 8 columns, as the decoder's dlogits
    are."""
    dev = cuda_device
    g = torch.Generator(device=dev).manual_seed(K + 7 * M + 13 * N)
    draw = lambda r, c: torch.randint(1, 3, (r, c), generator=g, device=dev, dtype=torch.uint8)
    buf = torch.zeros(K, (M + 7) // 8 * 8, device=dev, dtype=torch.bfloat16)
    dy = buf[:, :M]
    dy.copy_(draw(K, M))
    x = draw(K, N).to(torch.bfloat16)
    dw = torch.zeros(M, N, device=dev)
    engine._linear_wgrad(dy, x, dw)
    assert 4 * K < 2 ** 24
    exact = EB.gemm(dy.t(), x.t(), EB.U32, 0.0, block_k=BLOCK)[0]
    # distinct rows and distinct 128-column blocks (one output tile wide): a tile stored at another (m0, n0) shows
    assert torch.unique(exact, dim=0).shape[0] == M
    assert torch.unique(exact.view(M, N // 128, 128).transpose(0, 1).reshape(N // 128, -1), dim=0).shape[0] == N // 128
    splits, per = EB.splitk_launch(K, engine._wgrad_splits(K, M, N))
    assert torch.equal(dw.double(), exact), (f"{splits} splits of {per} k-blocks: "
                                             f"max |err| {(dw.double() - exact).abs().max().item()}")
