"""Times the fully Bayesian GP baseline `priors.fast_gp_mix.evaluate_` (csrc/gp_mcmc.cu, one launch per call).

    python tools/time_gp_mcmc.py [--reps 3] [--cpu-chains 2]

For each shape (B datasets, T rows, F features, every `step`-th prefix; data from `fast_gp_mix.get_batch`; 300 warmup
steps and 100 samples per chain, the reference's defaults):
  * end to end: `evaluate_()` between CUDA events (one warm-up call first), median of --reps calls;
  * kernel alone: `gp_mcmc_kernel` time from torch.profiler in a separate call;
  * work: leapfrog steps and mean tree depth from the diagnostics; fp64 FLOP counted as t^3 per potential evaluation
    (Cholesky, inverse and K^-1, t^3/3 each) over the kernel time, against the 34 TFLOP/s FP64 (non-tensor) H100 SXM
    data-sheet figure;
  * for contrast, the CPU NUTS restatement (oracle/gp_mcmc_oracle.py, one host thread) on --cpu-chains chains at the
    largest prefix, in seconds per chain.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from transformerscandobayesianinference_b200 import _lib as L  # noqa: E402
from transformerscandobayesianinference_b200.priors import fast_gp_mix  # noqa: E402

SHAPES = [(100, 50, 1, 1), (1000, 100, 1, 10), (100, 128, 5, 10)]     # B, T, F, prefix step
FP64_PEAK = 34e12
W, S = 300, 100


def card():
    if not torch.cuda.is_available():
        raise SystemExit("time_gp_mcmc needs a CUDA device (nothing is timed on the host alone)")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-chains", type=int, default=2)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    print(f"[time_gp_mcmc] card: {card()}", flush=True)
    col = {n: i for i, n in enumerate(L.GP_MCMC_DIAG_NAMES)}
    for B, T, F, step in SHAPES:
        torch.manual_seed(B + T + F)
        x, y, _ = fast_gp_mix.get_batch(B, T, F, device=dev)
        ts = list(range(1, T, step))
        # every prefix: evaluate_ itself; every step-th prefix: the launch evaluate_ makes, restricted to those prefixes
        xs, ys = x[:max(ts) + 1], y[:max(ts) + 1]

        def run():
            if step == 1:                                             # the public entry point itself
                return fast_gp_mix.evaluate_(xs, ys, ys, {}, device=dev, num_samples=S, warmup_steps=W, seed=1)
            xb, yb = xs.transpose(0, 1).contiguous(), ys.transpose(0, 1).contiguous()
            return fast_gp_mix.sample_posterior(xb, yb, ts, {}, S, W, seed=1)
        run()
        torch.cuda.synchronize()
        times = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / 1e3)
        xb, yb = xs.transpose(0, 1).contiguous(), ys.transpose(0, 1).contiguous()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            r = fast_gp_mix.sample_posterior(xb, yb, ts, {}, S, W, seed=1, trace=True)
            torch.cuda.synchronize()
        kern = sum(e.device_time for e in prof.events() if "gp_mcmc_kernel" in e.name and e.device_time > 0) / 1e6
        tt = torch.tensor(ts, dtype=torch.float64, device=dev).view(-1, 1)
        evals = r["diag"][..., col["evals"]].double()
        fl = float((evals * tt ** 3).sum())
        depth = r["trace"][..., F + 3]
        res = {"B": B, "T": T, "F": F, "prefixes": len(ts), "chains": len(ts) * B,
               "entry": "evaluate_" if step == 1 else "sample_posterior", "call_s": sorted(times), "kernel_s": kern,
               "mean_leapfrog_per_chain": float(r["diag"][..., col["leapfrog"]].double().mean()),
               "mean_evals_per_chain": float(evals.mean()), "mean_tree_depth": float(depth.mean()),
               "max_depth_hits": int(r["diag"][..., col["max_depth_hits"]].sum()),
               "div_sampling": int(r["diag"][..., col["div_sampling"]].sum()),
               "gflop": fl / 1e9, "tflops": fl / kern / 1e12 if kern > 0 else None,
               "share_of_fp64_peak": fl / kern / FP64_PEAK if kern > 0 else None}
        if args.cpu_chains > 0:
            from oracle import gp_mcmc_oracle as M
            t = ts[-1]
            xd, yd = xb.double().cpu().numpy(), yb.double().cpu().numpy()
            t0 = time.time()
            for b in range(args.cpu_chains):
                M.nuts_chain(M.potential_and_grad_np(xd[b, :t], yd[b, :t]), F + 2, S, W, 1, b=b, t=t)
            res.update({"cpu_restatement_t": t, "cpu_restatement_s_per_chain": (time.time() - t0) / args.cpu_chains})
        print(json.dumps(res), flush=True)
    print(f"[time_gp_mcmc] card (again): {card()}", flush=True)


if __name__ == "__main__":
    main()
