"""Time the learned-temperature decoder heads (decoders.ScaledDecoder, decoders.FixedScaledDecoder) against the default
decoder: forward + backward of the head alone at the BASELINE cfg-2 shape (batch 512, T = 1000, single_eval_pos 500, so
256 000 query rows; E = 512, nhid = 1024, 100 outputs), and the step time of `train()` with each head.

    python tools/time_decoders.py [--reps 20] [--train-steps 10]
"""
import argparse
import os
import random
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.gpu_timing import card, event_times  # noqa: E402
from transformerscandobayesianinference_b200 import (bar_distribution, decoders, encoders, engine, priors,  # noqa: E402
                                                     train as train_mod)

B, T, SEP, E, NHID, N_OUT = 512, 1000, 500, 512, 1024, 100


def head_times(reps):
    dev = torch.device("cuda:0")
    prec = engine.default_precision()
    hq = torch.randn((T - SEP) * B, E, device=dev).to(engine.act_dtype(prec)).requires_grad_()
    heads = {"default": torch.nn.Sequential(torch.nn.Linear(E, NHID), torch.nn.GELU(), torch.nn.Linear(NHID, N_OUT)),
             "ScaledDecoder": decoders.ScaledDecoder(E, NHID, N_OUT),
             "FixedScaledDecoder": decoders.FixedScaledDecoder(E, NHID, N_OUT)}
    gout = torch.randn(hq.shape[0], N_OUT, device=dev)
    out = {}
    random.seed(0)
    for name, m in heads.items():
        m.to(dev)
        if name == "default":
            run = lambda m=m: engine.DecoderFn.apply(hq, m[0].weight, m[0].bias, m[2].weight, m[2].bias, prec)
        else:
            run = lambda m=m: m.fused(hq, (hq.shape[0],), prec)

        def step(run=run):
            run().backward(gout)
        out[name] = event_times(step, reps, warmup=3)[reps // 2]
    return out


def train_step_times(steps):
    ys = priors.fast_gp.get_batch(500, T, 1, device="cuda:0")[1]
    crit = bar_distribution.FullSupportBarDistribution(bar_distribution.get_bucket_limits(N_OUT, ys=ys.cpu()))
    out = {}
    for name, dec in (("default", None), ("ScaledDecoder", decoders.ScaledDecoder),
                      ("FixedScaledDecoder", decoders.FixedScaledDecoder)):
        torch.manual_seed(0); random.seed(0)
        tr = train_mod.build_trainer(priors.fast_gp.DataLoader, crit, encoders.Linear, emsize=E, nhid=NHID, nlayers=6,
                                     nhead=4, dropout=0.0, epochs=1, steps_per_epoch=steps + 3, batch_size=B, bptt=T,
                                     lr=1e-4, warmup_epochs=0, y_encoder_generator=encoders.Linear, decoder=dec,
                                     single_eval_pos_gen=SEP, verbose=False,
                                     extra_prior_kwargs_dict={"num_features": 1, "hyperparameters": {
                                         "noise": 1e-4, "outputscale": 1.0, "lengthscale": .6}})
        x, y, tgt = priors.fast_gp.get_batch(B, T, 1, device="cuda:0", hyperparameters={
            "noise": 1e-4, "outputscale": 1.0, "lengthscale": .6})
        out[name] = event_times(lambda: tr.step((x, y), tgt, SEP), steps, warmup=3)[steps // 2]
        del tr
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--train-steps", type=int, default=10)
    args = ap.parse_args()
    print(card("time_decoders"))
    print(f"precision {engine.default_precision()}; head rows {(T - SEP) * B} (B {B}, T {T}, sep {SEP}), E {E}, "
          f"nhid {NHID}, n_out {N_OUT}; median of each sample set")
    for name, s in head_times(args.reps).items():
        print(f"head fwd+bwd  {name:20s} {s * 1e3:8.3f} ms")
    for name, s in train_step_times(args.train_steps).items():
        print(f"train step    {name:20s} {s * 1e3:8.3f} ms")


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"({time.time() - t0:.0f} s)")
