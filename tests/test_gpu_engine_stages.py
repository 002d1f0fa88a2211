"""The engine's training step op by op: every kernel call of embedding -> layers -> decoder -> loss -> backward is
recorded (oracle/engine_stages.Recorder), the call plan of the engine path is asserted, and every stage is held to its
kernel's per-element fp64 bound, with the exact value computed from the engine's own stored outputs of the earlier
stages chosen by their role in the reference layer.  This checks the wiring the per-kernel tests cannot see: which
tensor, mask and seed meet which gradient, the fused bias and delta paths, the bf16 weight copies, the gradient buckets."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L, bar_distribution, engine, optim, transformer
from oracle import engine_stages as ES
from oracle.make_golden import MODEL_CASES, CONFIG_CASES, build_case_weights, case_inputs, case_borders, case_targets


def _model(case, precision, p, dev):
    ctor = lambda enc, yenc: transformer.TransformerModel(enc, case["n_out"], case["E"], case["H"], case["nhid"],
                                                          case["L"], p, y_encoder=yenc)
    m = build_case_weights(ctor, case).to(dev)
    m.precision = precision
    m.train()
    return m


def _loss(m, case, x, y, dev, seed_key):
    """One forward and backward; returns the dropout seed TransformerModel.forward drew."""
    torch.manual_seed(seed_key)
    seed = int(torch.randint(0, 2 ** 31 - 1, (1,)).item())
    torch.manual_seed(seed_key)
    logits = m((x, y), single_eval_pos=case["sep"])
    t = case_targets(case, y)
    if case.get("head", "bar") == "bar":
        crit = bar_distribution.FullSupportBarDistribution(case_borders(case)).to(dev)
        loss = crit(logits.reshape(-1, case["n_out"]), t.flatten()).mean()
    else:
        loss = torch.nn.BCEWithLogitsLoss()(logits.flatten(), t.flatten())
    loss.backward()
    return seed


def _paths(precision, E, H):
    tc_attn = precision == "bf16" and E // H == 128
    fuse = tc_attn and engine._DELTA_FUSION
    return {"u_is_grad": precision == "bf16" and engine._GELU_GRAD_FWD, "rowdot": fuse, "tc_attn": tc_attn}


def _step_checked(m, case, precision, p, dev, tag, seed_key=1):
    """Run one recorded step of model m and check every stage; returns the checker (worst ratios per stage)."""
    x, y = (t.to(dev) for t in case_inputs(case))
    rec = ES.Recorder(L).install()
    try:
        seed = _loss(m, case, x, y, dev, seed_key)
    finally:
        rec.remove()
    torch.cuda.synchronize()
    thr = L.drop_threshold(p) if p else 0

    def mask(li, site, rows, cols):
        out = torch.empty(rows, cols, device=dev, dtype=torch.uint8)
        L.dropout_keep_mask(out, engine.site_seed(seed, li, site), thr)
        return out

    paths = _paths(precision, case["E"], case["H"])
    paths["fused_bias"] = paths.pop("tc_attn") and not thr
    chk = ES.StageCheck(T=case["T"], B=case["B"], H=case["H"], sep=case["sep"], thr=thr, mask=mask, num_sms=L.num_sms(),
                        paths=paths, tag=f"{tag}: ")
    layers = [dict(zip(ES.LAYER_PARAM_NAMES, [t.detach() for t in engine.layer_params(l)])) for l in m.transformer_encoder.layers]
    grads = [dict(zip(ES.LAYER_PARAM_NAMES, [t.grad for t in engine.layer_params(l)])) for l in m.transformer_encoder.layers]
    bar = case.get("head", "bar") == "bar"
    chk.step(rec.calls, x=x, y=y, emb=(m.encoder.weight.detach(), m.encoder.bias.detach(), m.y_encoder.weight.detach(),
                                       m.y_encoder.bias.detach()),
             layers=layers, dec=(m.decoder[0].weight.detach(), m.decoder[0].bias.detach(), m.decoder[2].weight.detach(),
                                 m.decoder[2].bias.detach()),
             precision=precision, borders=case_borders(case).to(dev) if bar else None, grads=grads)
    chk.report(tag)
    return chk


CASES = ([("dh128", "bf16", p, ab) for p in (0.0, 0.2) for ab in ("fused", "unfused")]
         + [("cfg1_small", "bf16", p, "fused") for p in (0.0, 0.5)]
         + [("sep0", "fp32", 0.0, "fused"), ("sep_last", "fp32", 0.2, "fused"), ("feat5_ragged", "fp32", 0.0, "fused")]
         + [(name, "bf16", 0.0, "fused") for name in CONFIG_CASES] + [("cfg2_b4", "bf16", 0.2, "fused")])


@pytest.mark.parametrize("name,precision,p,ab", CASES)
def test_engine_step_stages(cuda_device, monkeypatch, name, precision, p, ab):
    """bf16 head dim 128 (fused bias, fused delta, GELU' from the forward, and with both A/B switches off), bf16 head dim
    32 (wgmma GEMMs, SIMT attention), fp32 (everything SIMT), every BASELINE.json configuration shape."""
    case = MODEL_CASES.get(name) or CONFIG_CASES[name]
    if ab == "unfused":
        monkeypatch.setattr(engine, "_DELTA_FUSION", False)
        monkeypatch.setattr(engine, "_GELU_GRAD_FWD", False)
    m = _model(case, precision, p, cuda_device)
    _step_checked(m, case, precision, p, cuda_device, f"{name} {precision} p={p} {ab}")


def test_engine_stages_after_optimizer_step(cuda_device):
    """A second step after one FusedClipAdam update reads the optimizer's bf16 shadows; after an in-place edit of one
    weight the GEMMs must read a fresh cast, not the stale shadow (every weight operand equals bf16(master))."""
    case = MODEL_CASES["dh128"]
    m = _model(case, "bf16", 0.2, cuda_device)
    opt = optim.FusedClipAdam(m.parameters(), lr=1e-3, max_grad_norm=1.0)
    x, y = (t.to(cuda_device) for t in case_inputs(case))
    _loss(m, case, x, y, cuda_device, 3)
    opt.step()
    opt.zero_grad()
    w1 = m.transformer_encoder.layers[1].linear1.weight
    assert getattr(w1, "_pfn_shadow", None) is not None and w1._pfn_shadow[1] == w1._version
    _step_checked(m, case, "bf16", 0.2, cuda_device, "dh128 after Adam", seed_key=4)
    opt.step()
    opt.zero_grad()
    with torch.no_grad():
        w1.mul_(1.01)
    _step_checked(m, case, "bf16", 0.2, cuda_device, "dh128 after an in-place edit", seed_key=5)


@pytest.mark.parametrize("p", [0.0, 0.2])
def test_grad_buckets_are_final_when_reported(cuda_device, monkeypatch, p):
    """The data-parallel contract: each bucket handed to GRAD_BUCKET_HOOK is one layer's 12 gradients (the decoder's 4),
    and nothing writes them after it is reported (OverlappedGradReducer all-reduces the bucket in place at that moment)."""
    case = MODEL_CASES["dh128"]
    buckets = []
    monkeypatch.setattr(engine, "GRAD_BUCKET_HOOK", lambda flat: buckets.append(flat.clone()))
    monkeypatch.setattr(engine, "GRAD_BUCKET_SYNC", lambda: None)
    m = _model(case, "bf16", p, cuda_device)
    x, y = (t.to(cuda_device) for t in case_inputs(case))
    _loss(m, case, x, y, cuda_device, 6)
    torch.cuda.synchronize()
    layers = m.transformer_encoder.layers
    dec = [m.decoder[0].weight, m.decoder[0].bias, m.decoder[2].weight, m.decoder[2].bias]
    want = [dec] + [list(engine.layer_params(layers[li])) for li in reversed(range(len(layers)))]
    assert len(buckets) == len(want)
    for got, params in zip(buckets, want):
        final = torch.cat([t.grad.flatten() for t in params])
        assert got.numel() == final.numel() and torch.equal(got, final)
