"""Device time of the sklearn priors' baselines at the reference's __main__ shapes (B = 1000 datasets, T = 10, F = 10):
priors.ridge.evaluate(alpha=.01) (reference priors/ridge.py:37-39) and priors.gp.evaluate at length scale .6
(priors/gp.py:64-70), end to end (inputs on the device, the loss tensor on the host), with the card's name and power
limit read in the same run.  Next to them, when oracle/_ref holds the vendored reference (oracle/sklearn_priors_ref.py),
the reference's own sklearn loop on the host cores for the same inputs, on the first `--ref-datasets` datasets.

    python tools/time_regression_baselines.py [--reps 5] [--ref-datasets 100]
"""
import argparse
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from transformerscandobayesianinference_b200.priors import gp, ridge  # noqa: E402
from gpu_timing import card, event_times  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-datasets", type=int, default=100)
    a = ap.parse_args()
    print(f"card: {card('time_regression_baselines')}")
    torch.manual_seed(0)
    B, T, F = 1000, 10, 10
    rx, ry, ryn = (v.cuda() for v in ridge.get_batch(B, T, F, noisy_std=.01))
    gx, gy, _ = gp.get_batch(B, T, F, noisy_std=.6)
    for name, fn in (("ridge.evaluate(alpha=.01)", lambda: ridge.evaluate(rx, ry, ryn, alpha=.01)),
                     ("gp.evaluate(ls=.6, nll)", lambda: gp.evaluate(gx, gy, gy))):
        t = event_times(fn, a.reps)              # each call ends in a copy of the losses to the host
        best, med = t[0], t[len(t) // 2]
        print(f"{name:28s} B={B} T={T} F={F}: device {best * 1e3:8.2f} ms best, {med * 1e3:8.2f} ms median")
    if os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "sklearn_priors")):
        import warnings
        from oracle import sklearn_priors_ref
        ref_ridge, ref_gp = sklearn_priors_ref.load()
        n = a.ref_datasets
        warnings.simplefilter("ignore")
        for name, fn in (("reference ridge.evaluate", lambda: ref_ridge.evaluate(rx[:, :n].cpu(), ry[:, :n].cpu(),
                                                                                ryn[:, :n].cpu(), alpha=.01)),
                         ("reference gp.evaluate", lambda: ref_gp.evaluate(gx[:, :n].cpu(), gy[:, :n].cpu(),
                                                                          gy[:, :n].cpu()))):
            t0 = time.perf_counter()
            fn()
            s = time.perf_counter() - t0
            print(f"{name:28s} {n} of {B} datasets on {os.cpu_count()} host cores: {s:8.2f} s "
                  f"(x{B / n:.0f} for the batch: {s * B / n:8.1f} s)")
    else:
        print("reference: oracle/_ref/sklearn_priors absent, not run")


if __name__ == "__main__":
    main()
