"""Times the fitted-hyperparameter GP baseline `priors.fast_gp_mix.evaluate` (csrc/gp_fit.cu, one launch per call).

    python tools/time_gp_fit.py [--reps 3] [--scipy-datasets 2]

For each shape a user would run (B datasets, T rows, F features; data from `fast_gp_mix.get_batch`):
  * end to end: `evaluate()` between CUDA events (one warm-up call first), median of --reps calls;
  * kernel alone: `gp_fit_kernel` time from torch.profiler in a separate call;
  * work: fp64 FLOP counted from the returned evaluation counts, t^3 per objective evaluation (Cholesky t^3/3, inverse
    t^3/3, K^-1 t^3/3; the gradient's O(t^2 F) is left out), over the kernel time, against the 34 TFLOP/s FP64
    (non-tensor) H100 SXM data-sheet figure;
  * for contrast, the scipy restatement (oracle/gp_fit_oracle.py, L-BFGS-B on the host cores, one process per core) on
    --scipy-datasets datasets at every 10th prefix, extrapolated per call.  botorch itself is not run.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import multiprocessing as mp
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from transformerscandobayesianinference_b200.priors import fast_gp_mix  # noqa: E402
from gpu_timing import card, event_times, kernel_seconds  # noqa: E402

SHAPES = [(1000, 100, 1), (1000, 100, 5), (100, 128, 5)]
FP64_PEAK = 34e12


def flops(r, ts):
    t = torch.tensor(ts, dtype=torch.float64, device=r["nevals"].device).view(-1, 1)
    return float(((r["nevals"].double() + 1.0) * t ** 3).sum())      # +1: the final evaluation at the returned point


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--scipy-datasets", type=int, default=2)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    print(f"[time_gp_fit] card: {card('time_gp_fit')}", flush=True)
    results = []
    for B, T, F in SHAPES:
        torch.manual_seed(B + T + F)
        x, y, _ = fast_gp_mix.get_batch(B, T, F, device=dev)
        losses, _, _ = fast_gp_mix.evaluate(x, y, y, device=dev)    # warm-up (module load, first launch)
        times = event_times(lambda: fast_gp_mix.evaluate(x, y, y, device=dev), args.reps, warmup=0)
        ts = list(range(1, T))
        xb, yb = x.transpose(0, 1).contiguous(), y.transpose(0, 1).contiguous()
        r = fast_gp_mix.fit_map(xb, yb, ts, {})
        kernels = kernel_seconds(lambda: fast_gp_mix.fit_map(xb, yb, ts, {}))
        kern = sum(s for name, (s, _) in kernels.items() if "gp_fit_kernel" in name)
        fl = flops(r, ts)
        st = r["status"]
        res = {"B": B, "T": T, "F": F, "evaluate_s": times, "kernel_s": kern, "gflop": fl / 1e9,
               "tflops": fl / kern / 1e12 if kern > 0 else None,
               "share_of_fp64_peak": fl / kern / FP64_PEAK if kern > 0 else None,
               "mean_evals": float(r["nevals"].double().mean()), "max_evals": int(r["nevals"].max()),
               "mean_iters": float(r["iters"].double().mean()),
               "status": {n: int((st == c).sum()) for c, n in fast_gp_mix._STATUS_NAMES.items()},
               "mean_nll": float(losses.double().mean())}
        if args.scipy_datasets > 0:
            from oracle import gp_fit_oracle as G
            xd, yd = xb.double().cpu(), yb.double().cpu()
            sub = ts[::10]
            jobs = [(xd[b, :t], yd[b, :t], xd[b, t]) for b in range(args.scipy_datasets) for t in sub]
            t0 = time.time()
            with mp.get_context("spawn").Pool(os.cpu_count()) as pool:
                pool.map(G.gp_fit_ref_job, jobs, chunksize=1)
            host = time.time() - t0
            per_dataset = host / args.scipy_datasets * len(ts) / len(sub)
            res.update({"scipy_restatement_cores": os.cpu_count(), "scipy_restatement_s_subset": host,
                        "scipy_restatement_fits": len(jobs),
                        "scipy_restatement_s_per_call_extrapolated": per_dataset * B})
        print(json.dumps(res), flush=True)
        results.append(res)
    print(f"[time_gp_fit] card (again): {card('time_gp_fit')}", flush=True)


if __name__ == "__main__":
    main()
