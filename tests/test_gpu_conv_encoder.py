"""encoders.Conv on the H100: each kernel of csrc/conv_encoder.cu against its per-element fp64 bound (oracle/conv_oracle.py)
fed the oracle's own inputs, the module's forward and gradients against the fp64 module, its bitwise properties, and
BASELINE configuration 5 (Omniglot 5-way 1-shot, conv encoder + 4-layer transformer, batch 256) through the trainer."""
import math

import pytest
import torch

from oracle import conv_oracle as co
from oracle import error_budget as eb
from transformerscandobayesianinference_b200 import _lib as L
from transformerscandobayesianinference_b200 import encoders, engine

pytestmark = pytest.mark.gpu
DEV = "cuda"
# (S, N): sides from the smallest to the largest image, one, a few and a configuration-5 batch of images.  Most output
# counts M = N (S - 2)^2 leave a partial last 128-pixel tile, and a tile spans several images at the small sides and a
# few rows at the large ones
CASES = [(4, 1536), (5, 3), (6, 1536), (9, 3), (28, 1536), (33, 3), (105, 1), (112, 1)]
PRECISIONS = ["bf16", "fp32"]
IMG_BLOCK = 96          # images per fp64 oracle call (the im2col view of 1536 images at S = 28 is 1 M x 577)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _act(N, s, dt, gen, scale=1.0):
    """A post-ReLU activation: about half the entries exactly 0."""
    return torch.relu(torch.randn(N, s, s, 64, device=DEV, generator=gen) * scale).to(dt)


def _weights(cin, gen):
    bound = 1.0 / math.sqrt(9 * cin)
    W = (torch.rand(64, cin, 3, 3, device=DEV, generator=gen) * 2 - 1) * bound
    b = (torch.rand(64, device=DEV, generator=gen) * 2 - 1) * bound
    return W, b


def _u(dt):
    return eb.U if dt == torch.bfloat16 else eb.U32


def _check_blocks(name, got, fn, c, N):
    worst = 0.0
    for n0 in range(0, N, IMG_BLOCK):
        exact, bound = fn(slice(n0, n0 + IMG_BLOCK))
        worst = max(worst, eb.check(f"{name} [{n0}:]", got[n0:n0 + IMG_BLOCK], exact, bound, c, verbose=False))
    print(f"[error-budget] {name}: worst err/bound = {worst:.4g} (c = {c})")


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("S,N", CASES)
def test_conv_fwd_kernels(S, N, precision):
    dt = engine.act_dtype(precision)
    gen = _gen(S * 7 + N)
    x = torch.rand(N, S, S, device=DEV, generator=gen)
    W1, b1 = _weights(1, gen)
    y = torch.full((N, S - 2, S - 2, 64), float("nan"), device=DEV, dtype=dt)
    L.conv_fwd(x, W1, b1, y, N, S, 1)
    _check_blocks(f"conv_fwd C_in=1 S={S} N={N} {precision}", y,
                  lambda sl: co.conv_fwd(x[sl, :, :, None], W1, b1, _u(dt), co.C_ACC_CONV_DIRECT), co.C_CONV, N)
    s = S - 2
    if s < 4:
        return
    xa = _act(N, s, dt, gen)
    W, b = _weights(64, gen)
    w_op = engine.conv_weight_operand(W) if dt == torch.bfloat16 else W
    y2 = torch.full((N, s - 2, s - 2, 64), float("nan"), device=DEV, dtype=dt)
    L.conv_fwd(xa, w_op, b, y2, N, s, 64)
    Wk = W.to(dt).float() if dt == torch.bfloat16 else W      # the kernel's own (bf16-cast) weights
    c_acc = co.C_ACC_CONV if dt == torch.bfloat16 else co.C_ACC_CONV_DIRECT
    _check_blocks(f"conv_fwd C_in=64 S={s} N={N} {precision}", y2,
                  lambda sl: co.conv_fwd(xa[sl], Wk, b, _u(dt), c_acc), co.C_CONV, N)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("S,N", CASES)
def test_conv_dgrad_kernel(S, N, precision):
    s = S - 2                    # the 64 -> 64 layer whose input side is S - 2 (the second conv)
    if s < 4:
        pytest.skip("one conv only: no data gradient")
    dt = engine.act_dtype(precision)
    gen = _gen(S * 11 + N)
    x = _act(N, s, dt, gen)
    W, _ = _weights(64, gen)
    gpad = torch.zeros(N, s + 2, s + 2, 64, device=DEV, dtype=dt)
    gpad[:, 2:s, 2:s] = (torch.randn(N, s - 2, s - 2, 64, device=DEV, generator=gen) * 1e-3).to(dt)
    out = torch.full((N, s + 4, s + 4, 64), float("nan"), device=DEV, dtype=dt)     # the kernel writes the border too
    w_op = engine.conv_weight_operand(W, dgrad=True) if dt == torch.bfloat16 else W
    L.conv_dgrad(gpad, w_op, x, out, N, s)
    Wk = W.to(dt).float() if dt == torch.bfloat16 else W
    assert (out[:, :2] == 0).all() and (out[:, -2:] == 0).all() and (out[:, :, :2] == 0).all() and (out[:, :, -2:] == 0).all()
    _check_blocks(f"conv_dgrad S={s} N={N} {precision}", out[:, 2:-2, 2:-2],
                  lambda sl: co.conv_dgrad(gpad[sl], Wk, x[sl], _u(dt),
                                           co.C_ACC_CONV if dt == torch.bfloat16 else co.C_ACC_CONV_DIRECT), co.C_CONV, N)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("S,N", CASES)
def test_conv_wgrad_kernels(S, N, precision):
    dt = engine.act_dtype(precision)
    gen = _gen(S * 13 + N)
    layers = [(S, 1)] + ([(S - 2, 64)] if S - 2 >= 4 else [])
    for s, cin in layers:
        x = torch.rand(N, s, s, device=DEV, generator=gen) if cin == 1 else _act(N, s, dt, gen)
        g = torch.zeros(N, s + 2, s + 2, 64, device=DEV, dtype=dt)
        g[:, 2:s, 2:s] = (torch.randn(N, s - 2, s - 2, 64, device=DEV, generator=gen) * 1e-3).to(dt)
        dw = torch.full((64, cin, 3, 3), float("nan"), device=DEV)
        db = torch.full((64,), float("nan"), device=DEV)
        L.conv_wgrad(g, x, dw, db, N, s, cin)
        ew, eb_, bw, bb = co.conv_wgrad(g[:, 2:s, 2:s], x if cin == 64 else x[..., None])
        tag = f"C_in={cin} S={s} N={N} {precision}"
        eb.check(f"conv_wgrad dW {tag}", dw, ew, bw, 1.0)
        eb.check(f"conv_wgrad db {tag}", db, eb_, bb, 1.0)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("s,N", [(2, 1536), (1, 3), (3, 3), (4, 1), (8, 1536), (107, 1)])
def test_conv_mean_kernels(s, N, precision):
    dt = engine.act_dtype(precision)
    gen = _gen(s * 17 + N)
    y = _act(N, s, dt, gen)
    feat = torch.full((N, 64), float("nan"), device=DEV, dtype=dt)
    L.conv_mean_fwd(y, feat, N, s)
    eb.check(f"conv_mean_fwd s={s} N={N} {precision}", feat, *co.mean_fwd(y, _u(dt)), co.C_MEAN)
    dfeat = torch.randn(N, 64, device=DEV, generator=gen).to(dt)
    g = torch.full((N, s + 4, s + 4, 64), float("nan"), device=DEV, dtype=dt)         # the kernel writes the border too
    L.conv_mean_bwd(dfeat, y, g, N, s)
    eb.check(f"conv_mean_bwd s={s} N={N} {precision}", g[:, 2:s + 2, 2:s + 2], *co.mean_bwd(dfeat, y, _u(dt)), co.C_MEAN)
    assert (g[:, :2] == 0).all() and (g[:, -2:] == 0).all() and (g[:, :, :2] == 0).all() and (g[:, :, -2:] == 0).all()


# tolerances of the whole module against fp64: relative Frobenius-norm error of the output and of each gradient
MODULE_TOL = {"bf16": 3e-2, "fp32": 1e-4}


def _module(S, E, precision, seed=0):
    torch.manual_seed(seed)
    m = encoders.Conv(S * S, E)
    m.precision = precision
    return m.to(DEV)


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300)).item()


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("S,N", [(4, 64), (6, 3), (9, 17), (28, 256), (33, 3), (112, 2)])
def test_module_forward_and_gradients(S, N, precision):
    m = _module(S, 96, precision)
    gen = _gen(S + N)
    x = torch.rand(N, S * S, device=DEV, generator=gen)
    dout = torch.randn(N, 96, device=DEV, generator=gen)
    out = m(x)
    out.backward(dout)
    params = [p for c in m.convs[:m.n_conv] for p in (c.weight, c.bias)] + [m.linear.weight, m.linear.bias]
    ref_out, ref_grads = co.gradients(x, params, S, dout)
    tol = MODULE_TOL[precision]
    errs = {"out": _rel(out, ref_out)}
    for i, (p, r) in enumerate(zip(params, ref_grads)):
        errs[f"grad{i}"] = _rel(p.grad, r)
    print(f"[conv-module] S={S} N={N} {precision}: " + ", ".join(f"{k} {v:.3g}" for k, v in errs.items()))
    assert all(v <= tol for v in errs.values()), errs
    for c in m.convs[m.n_conv:]:
        assert c.weight.grad is None and c.bias.grad is None


def _run(m, x, dout):
    m.zero_grad(set_to_none=True)
    out = m(x)
    out.backward(dout)
    return out.detach().clone(), {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}


def _same(a, b, tag):
    (out1, g1), (out2, g2) = a, b
    assert torch.equal(out1, out2), f"{tag}: outputs differ"
    assert g1.keys() == g2.keys()
    for k in g1:
        assert torch.equal(g1[k], g2[k]), f"{tag}: {k} differs"


@pytest.mark.parametrize("precision", PRECISIONS)
def test_module_bitwise_properties(precision):
    S, N = 28, 300
    m = _module(S, 64, precision)
    gen = _gen(5)
    x = torch.rand(N, S * S, device=DEV, generator=gen)
    dout = torch.randn(N, 64, device=DEV, generator=gen)
    first = _run(m, x, dout)
    _same(first, _run(m, x, dout), "second run")
    with torch.no_grad():
        alone = m(x[137:138])
    assert torch.equal(alone, first[0][137:138])
    # NaN-prefilled allocations: every element the kernels' outputs are read from is written
    torch.cuda.empty_cache()
    junk = torch.full((1 << 28,), float("nan"), device=DEV)
    del junk
    _same(first, _run(m, x, dout), "NaN-prefilled memory")


def test_unused_convs_get_no_gradient():
    m = _module(6, 32, "bf16")
    x = torch.rand(4, 36, device=DEV)
    m(x).sum().backward()
    assert m.n_conv == 2
    assert all(c.weight.grad is not None for c in m.convs[:2])
    assert all(c.weight.grad is None and c.bias.grad is None for c in m.convs[2:])


def test_module_rejects_input_gradient_on_gpu():
    m = _module(28, 32, "bf16")
    with pytest.raises(ValueError):
        m(torch.rand(2, 784, device=DEV, requires_grad=True))


# ---------------------------------------------------------------------------------------------------------------------
# BASELINE configuration 5
# ---------------------------------------------------------------------------------------------------------------------
def synthetic_bank(S=28, seed=0):
    """Omniglot-shaped bank (1623 characters x 20 images, uint8, 255 = background; 964 background and 659 evaluation
    characters) whose 20 images of a character share one ink pattern up to noise."""
    import numpy as np
    from transformerscandobayesianinference_b200.priors import omniglot
    rng = np.random.default_rng(seed)
    ink = (rng.random((1623, 1, S, S)) < 0.15) ^ (rng.random((1623, 20, S, S)) < 0.03)
    return omniglot.Bank(np.where(ink, 0, 255).astype(np.uint8), [("background", 0, 964), ("evaluation", 964, 659)])


def _episodes(bank, B, seed):
    from transformerscandobayesianinference_b200.priors import omniglot
    return omniglot.sample_episodes(bank, omniglot.episode_desc(bank, B, 5, 1), seed=seed)


CFG5 = dict(emsize=512, nhid=1024, nlayers=4, nhead=4, dropout=0.0, bptt=6, warmup_epochs=0,
            y_encoder_generator=encoders.get_Canonical(5), single_eval_pos_gen=5,
            extra_prior_kwargs_dict=dict(num_features=784, num_outputs=5))


@pytest.fixture
def cfg5_bank(monkeypatch):
    """priors.omniglot.DataLoader reads its bank through `load_bank`; serve the synthetic one."""
    from transformerscandobayesianinference_b200.priors import omniglot
    bank = synthetic_bank()
    monkeypatch.setattr(omniglot, "load_bank", lambda S, root="omniglot": bank)
    return bank


def _encoder_params(enc):
    return [p for c in enc.convs[:enc.n_conv] for p in (c.weight, c.bias)] + [enc.linear.weight, enc.linear.bias]


def test_cfg5_trainer_step_and_encoder_gradients(cfg5_bank):
    """train(priors.omniglot.DataLoader, CE, encoders.Conv, ...) at BASELINE configuration 5: one Trainer.step at T = 6,
    B = 256, sep 5 (aggregate_k_gradients = 2 keeps the step's gradients: the optimizer steps on the second call)."""
    from transformerscandobayesianinference_b200.priors import omniglot
    from transformerscandobayesianinference_b200.train import build_trainer
    torch.manual_seed(0)
    tr = build_trainer(omniglot.DataLoader, torch.nn.CrossEntropyLoss(reduction="none"), encoders.Conv, epochs=1,
                       steps_per_epoch=2, batch_size=256, lr=1e-4, aggregate_k_gradients=2, **CFG5)
    enc = tr.model.encoder
    assert isinstance(enc, encoders.Conv) and enc.n_conv == 5
    (x, y), target = next(iter(tr.dl))
    assert x.shape == (6, 256, 784)
    captured = {}

    def keep_output(mod, inp, o):
        o.retain_grad()
        captured["out"] = o
    h = enc.register_forward_hook(keep_output)
    loss, losses = tr.step((x, y), target, 5)
    h.remove()
    assert losses.shape == (1, 256) and torch.isfinite(loss)
    # the encoder's gradients against the fp64 oracle on the same batch and the encoder's output gradient of this step
    params = _encoder_params(enc)
    _, ref = co.gradients(x.reshape(-1, 784), params, 28, captured["out"].grad.reshape(-1, 512))
    errs = [_rel(p.grad, r) for p, r in zip(params, ref)]
    print(f"[conv-cfg5] Trainer.step loss {loss.item():.4f}, encoder gradient errors " + ", ".join(f"{e:.3g}" for e in errs))
    assert max(errs) <= MODULE_TOL["bf16"], errs


def _eval_loss(model, batches):
    model = model.to(DEV).eval()
    with torch.no_grad():
        return sum(torch.nn.functional.cross_entropy(model((x, y), single_eval_pos=5).reshape(-1, 5),
                                                     t[5:].reshape(-1)).item() for x, y, t in batches) / len(batches)


def test_cfg5_short_train_lowers_the_loss(cfg5_bank):
    """A short train() over the Omniglot DataLoader with encoders.Conv (fused clip + Adam, bf16 weight shadows) lowers the
    loss on held-out episodes of the synthetic bank (300 steps: 1.628 -> 1.615 on an H100; ln 5 = 1.609 is chance)."""
    from transformerscandobayesianinference_b200.priors import omniglot
    from transformerscandobayesianinference_b200.train import Losses, build_trainer, train
    kw = dict(CFG5, emsize=256, nhid=512)
    torch.manual_seed(0)
    start = build_trainer(omniglot.DataLoader, Losses.ce, encoders.Conv, epochs=1, steps_per_epoch=1, batch_size=64,
                          lr=1e-3, **kw).model
    state = {k: v.detach().clone() for k, v in start.state_dict().items()}
    held_out = [_episodes(cfg5_bank, 128, seed=10_000 + i) for i in range(4)]
    before = _eval_loss(start, held_out)
    torch.manual_seed(1)
    total_loss, _, model = train(omniglot.DataLoader, Losses.ce, encoders.Conv, epochs=1, steps_per_epoch=300,
                                 batch_size=64, lr=1e-3, load_weights_from_this_state_dict=state, verbose=False, **kw)
    after = _eval_loss(model, held_out)
    print(f"[conv-cfg5] train(): held-out loss {before:.4f} -> {after:.4f} (last epoch {total_loss:.4f})")
    assert math.isfinite(total_loss) and after < before - 0.005
