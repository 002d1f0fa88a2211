"""Robustness run of the other BASELINE.json configurations at full size on one GPU (parity is covered by the tests; this
checks that the full-size shapes run, are finite and learn-able, and reports time and peak memory).
  cfg4: priors.fast_gp_mix, T=2000, B=512 per GPU, E=512, 6 layers, sep=1000
  cfg3: priors.mlp (18 features), T=512, B=512, E=512, 12 layers, sep=256"""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from transformerscandobayesianinference_b200 import priors, bar_distribution, transformer, encoders

dev = torch.device("cuda:0")
bar_distribution.BarDistribution.defer_support_check = True


def run(name, get_batch, T, B, F, L, sep, steps=3, bce=False, **kw):
    torch.manual_seed(0)
    n_out = 1 if bce else 100
    model = transformer.TransformerModel(encoders.Linear(F, 512), n_out, 512, 4, 1024, L, 0.0, y_encoder=encoders.Linear(1, 512)).to(dev)
    if bce:
        bcel = torch.nn.BCEWithLogitsLoss(reduction='none')
        crit = lambda lg, tg: bcel(lg.flatten(), tg)
    else:
        ys = get_batch(64, T, F, device=str(dev), **kw)[1]
        crit = bar_distribution.FullSupportBarDistribution(bar_distribution.get_bucket_limits(100, ys=ys.float().cpu())).to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=1e-4, fused=True)
    torch.cuda.reset_peak_memory_stats()
    losses, times = [], []
    for s in range(steps):
        torch.cuda.synchronize(); t0 = time.time()
        x, y, tgt = get_batch(B, T, F, device=str(dev), **kw)
        logits = model((x, y), single_eval_pos=sep)
        loss = crit(logits.reshape(-1, n_out), tgt[sep:].flatten()).mean()
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 1.)
        opt.step(); opt.zero_grad(set_to_none=True)
        torch.cuda.synchronize(); times.append(time.time() - t0); losses.append(loss.item())
    assert all(l == l and abs(l) < 1e4 for l in losses), losses
    print(f"{name}: losses {[round(l, 4) for l in losses]}  step {min(times) * 1e3:.1f} ms  ({B / min(times):.0f} seq/s)  "
          f"peak mem {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB", flush=True)


which = sys.argv[1:] or ["cfg4", "cfg3"]
if "cfg4" in which:
    run("cfg4 fast_gp_mix T=2000 B=512 L=6", priors.fast_gp_mix.get_batch, 2000, 512, 1, 6, 1000, batch_size_per_gp_sample=64)
if "cfg3" in which:
    su = priors.utils     # the shipped bnn config (TabularEvalSimple.ipynb:154-176)
    hp = (lambda: 3, su.scaled_beta_sampler_f(2, 4, 150, 2), torch.nn.Tanh, su.gamma_sampler_f(3.62, .0677),
          su.gamma_sampler_f(1.87, .0528), lambda: 0.0, True, su.scaled_beta_sampler_f(1, 1.6, 18, 2), None, False, None,
          None, None, True, True, lambda n: ([], []), 0.0)
    run("cfg3 mlp prior T=512 B=512 F=18 L=12 BCE", priors.mlp.get_batch, 512, 512, 18, 12, 256, bce=True,
        hyperparameters=hp, batch_size_per_gp_sample=8)
