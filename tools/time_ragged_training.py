"""Time training with one single_eval_pos per dataset at the cfg2 shape (priors.fast_gp, T 1000, emsize 512, 4 heads,
6 layers, nhid 1024, bar head of 100 buckets, batch 512):

  step      Trainer.step (forward, masked bar-NLL, backward, fused Adam) with per-dataset values drawn by
            utils.per_dataset_sampler(get_weighted_single_eval_pos_sampler(T), batch), against the scalar step at the
            single_eval_pos that leaves the same mean number of query rows per dataset
  attention the ragged attention backward (_lib_ragged_train) on those values against the uniform backward at that
            scalar value, and the ragged backward with every value equal to it (what the ragged support costs by itself);
            each with its kernels' device times from torch.profiler in a pass of its own

    python tools/time_ragged_training.py [--reps 7] [--seed 0]
"""
import argparse
import os
import random
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.gpu_timing import card, event_times, kernel_seconds  # noqa: E402
from transformerscandobayesianinference_b200 import (_lib as L, _lib_ragged_train as LRT, bar_distribution,  # noqa: E402
                                                     encoders, priors, train as train_mod, utils)

T, B, E, H, NHID, NL, BARS = 1000, 512, 512, 4, 1024, 6, 100


def _trainer():
    ys = priors.fast_gp.get_batch(64, T, 1, device="cuda")[1]
    crit = bar_distribution.FullSupportBarDistribution(bar_distribution.get_bucket_limits(BARS, ys=ys.cpu()))
    return train_mod.build_trainer(priors.fast_gp.DataLoader, crit, encoders.Linear, emsize=E, nhid=NHID, nlayers=NL,
                                   nhead=H, dropout=0.0, epochs=1, steps_per_epoch=1, batch_size=B, bptt=T, lr=1e-4,
                                   warmup_epochs=0, y_encoder_generator=encoders.Linear,
                                   extra_prior_kwargs_dict={"num_features": 1}, single_eval_pos_gen=lambda: 0,
                                   verbose=False)


def _attention_bwd(seps, ragged, reps):
    dh = E // H
    g = torch.Generator(device="cuda").manual_seed(1)
    qkv = torch.randn(T * B, 3 * E, device="cuda", generator=g).to(torch.bfloat16)
    dout = torch.randn(T * B, E, device="cuda", generator=g).to(torch.bfloat16)
    out = torch.empty(T * B, E, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(B * H, T, device="cuda")
    dqkv, delta = torch.empty_like(qkv), torch.empty(B * H, T, device="cuda")
    if ragged:
        n_keys = torch.tensor(seps, dtype=torch.int32, device="cuda")
        LRT.attention_ragged_train_fwd(qkv, out, lse, T, B, H, dh, max(seps), n_keys)
        fn = lambda: LRT.attention_ragged_train_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, dh, max(seps), n_keys)
    else:
        L.attention_fwd(qkv, out, lse, T, B, H, dh, seps)
        fn = lambda: L.attention_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, dh, seps)
    kernels = {k: v for k, v in kernel_seconds(fn).items() if "attn_bwd" in k}
    return event_times(fn, reps, warmup=2), kernels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    print(card("time_ragged_training"))
    random.seed(args.seed)
    torch.manual_seed(args.seed)
    seps = utils.per_dataset_sampler(utils.get_weighted_single_eval_pos_sampler(T), B)()
    mean_q = sum(T - s for s in seps) / B
    scalar = T - round(mean_q)
    print(f"cfg2 shape: T {T}, batch {B}, emsize {E}, {H} heads, {NL} layers; weighted per-dataset values "
          f"{min(seps)}..{max(seps)}, mean query rows {mean_q:.1f}; scalar single_eval_pos {scalar}; "
          f"median of {args.reps} samples, each one CUDA-event bracket")
    med = lambda ts: ts[len(ts) // 2]
    tr = _trainer()
    x, y, _ = priors.fast_gp.get_batch(B, T, 1, device="cuda")
    data, targets = (x, y), y
    for name, sep in (("step, scalar", scalar), ("step, per-dataset", seps)):
        ts = event_times(lambda: tr.step(data, targets, sep), args.reps, warmup=2)
        print(f"  {name:34s} {med(ts) * 1e3:9.2f} ms   (min {ts[0] * 1e3:.2f}, max {ts[-1] * 1e3:.2f})")
    del tr
    torch.cuda.empty_cache()
    for name, sep, ragged in (("attention bwd, uniform scalar", scalar, False),
                              ("attention bwd, ragged all equal", [scalar] * B, True),
                              ("attention bwd, ragged per-dataset", seps, True)):
        ts, kernels = _attention_bwd(sep, ragged, args.reps)
        print(f"  {name:34s} {med(ts) * 1e3:9.2f} ms   (min {ts[0] * 1e3:.2f}, max {ts[-1] * 1e3:.2f})")
        for k, (sec, n) in sorted(kernels.items()):
            print(f"      {k[:70]:70s} {sec * 1e3:8.3f} ms")
        torch.cuda.empty_cache()


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"({time.time() - t0:.0f} s)")
