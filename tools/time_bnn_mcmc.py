"""Times the Bayesian-NN experiment's device paths: the NUTS baseline `eval_mcmc` (csrc/bnn_mcmc.cu, one launch per call)
and the prior `priors.pyro.get_batch` (csrc/bnn_prior.cu).

    python tools/time_bnn_mcmc.py [--reps 3] [--cpu-chains 1] [--no-sweep]

The reference's workloads: the `small` (F = 3, E = 5, d = 32) and `big` (F = 8, E = 64, d = 706) models, 100 datasets of
300 rows from `generate_toy_data`, 100 training rows, warmup = samples in {64, 512}; and the `training_samples` sweep
(training rows 2, 7, .., 97 at 512 / 512, one call each).  For every call: seconds between CUDA events (one warm-up call
first, the sorted times of --reps calls), and from the diagnostics of a traced call the leapfrog steps, mean tree depth,
depth-cap hits and divergences per chain.  Then `get_batch` at the notebook's batch (256 datasets of 300 rows), and the
CPU NUTS restatement (oracle/gp_mcmc_oracle.nuts_chain on oracle/bnn_oracle's potential, one host thread) at 64 / 64 in
seconds per chain.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from transformerscandobayesianinference_b200 import _lib as L  # noqa: E402
from transformerscandobayesianinference_b200 import mcmc_svi_transformer_on_bayesian as M  # noqa: E402
from transformerscandobayesianinference_b200.priors import pyro as P  # noqa: E402
from gpu_timing import card, event_times  # noqa: E402


def work(X, y, spec, n, steps):
    """Per-chain work of one call, from the kernel's diagnostics and trace."""
    col = {k: i for i, k in enumerate(L.GP_MCMC_DIAG_NAMES)}
    r = M.sample_bnn_posterior(X[:, :n], y[:, :n], X[:, n:], spec, steps, steps, seed=1, trace=True)
    diag, N = r["diag"].double(), X.shape[0]
    return {"leapfrog_per_chain": float(diag[:, col["leapfrog"]].mean()), "mean_tree_depth": float(r["trace"][..., -1].mean()),
            "depth_cap_hits_per_chain": float(diag[:, col["max_depth_hits"]].mean()),
            "div_warmup_per_chain": float(diag[:, col["div_warmup"]].mean()),
            "div_sampling_per_chain": float(diag[:, col["div_sampling"]].mean()),
            "mean_accept": float(r["accept"].mean()), "workspace_doubles_per_chain":
            L.bnn_mcmc_workspace(L.bnn_mcmc_desc(N, n, X.shape[1] - n, spec['num_features'], spec['embed'], steps, steps, 1))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-chains", type=int, default=1)
    ap.add_argument("--no-sweep", action="store_true")
    args = ap.parse_args()
    print(f"[time_bnn_mcmc] card: {card('time_bnn_mcmc')}", flush=True)
    dev = torch.device("cuda:0")
    for size in ("small", "big"):
        spec = M.get_default_model_spec(size)
        sampler = lambda: M.BayesianModel(spec, device="cuda:0")
        X, y = M.generate_toy_data(sampler(), spec["seq_len"], device=dev)
        d = spec["embed"] * spec["num_features"] + 3 * spec["embed"] + 2
        for steps in (64, 512):
            t = event_times(lambda: M.eval_mcmc(X, y, dev, sampler, 100, steps, steps, seed=1), args.reps)
            print(json.dumps(dict({"model": size, "d": d, "chains": 100, "train_rows": 100, "warmup": steps, "samples": steps,
                                   "eval_mcmc_s": t}, **work(X, y, spec, 100, steps))), flush=True)
        if not args.no_sweep:
            points = M.get_default_evaluation_points()
            M.eval_mcmc(X, y, dev, sampler, points[0], 8, 8, seed=1)
            per_point = [round(event_times(lambda: M.eval_mcmc(X, y, dev, sampler, n, 512, 512, seed=1), 1, warmup=0)[0], 3)
                         for n in points]
            print(json.dumps({"model": size, "sweep_train_rows": points, "warmup": 512, "samples": 512,
                              "eval_mcmc_s_per_point": per_point, "sweep_total_s": sum(per_point)}), flush=True)
        t = event_times(lambda: P.get_batch(256, 300, model=sampler, device=dev), max(args.reps, 10))
        print(json.dumps({"model": size, "get_batch": [256, 300], "get_batch_s": t}), flush=True)
        if args.cpu_chains > 0:
            from oracle import bnn_oracle as O
            Xd, yd = X[:, :100].double().cpu().numpy(), y[:, :100].cpu().numpy()
            t0 = time.time()
            for b in range(args.cpu_chains):
                O.bnn_chain_job((Xd[b], yd[b], spec["num_features"], spec["embed"], 64, 64, 1, b, 10))
            print(json.dumps({"model": size, "cpu_restatement_warmup_samples": [64, 64],
                              "cpu_restatement_s_per_chain": (time.time() - t0) / args.cpu_chains}), flush=True)
    print(f"[time_bnn_mcmc] card (again): {card('time_bnn_mcmc')}", flush=True)


if __name__ == "__main__":
    main()
