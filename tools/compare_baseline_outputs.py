"""Checks that two builds of the library give bitwise equal results for the GP and Bayesian-NN baselines: the MAP fit
(`priors.fast_gp_mix.fit_map`), the GP NUTS sampler (`fast_gp_mix.sample_posterior`) and the Bayesian-NN NUTS sampler
(`mcmc_svi_transformer_on_bayesian.sample_bnn_posterior`).

Used when csrc/gp_fit.cu, gp_mcmc.cu, bnn_mcmc.cu or the headers they share change without meaning to change results,
e.g. to compare the tree against its parent commit on a GPU:

    git worktree add /tmp/parent HEAD~1 && (cd /tmp/parent && python -m transformerscandobayesianinference_b200.csrc.build)
    python tools/compare_baseline_outputs.py run /tmp/old.pt --tree /tmp/parent
    python tools/compare_baseline_outputs.py run /tmp/new.pt
    python tools/compare_baseline_outputs.py compare /tmp/old.pt /tmp/new.pt

`run` imports the package (and its library) from --tree (default: this checkout) and saves every output tensor of seeded
calls: the fit at four shapes (theta, f, grad, mean, var, iters, nevals, status); the GP sampler at the sizes
tools/time_gp_mcmc.py times plus one run capped at tree depth 2; the Bayesian-NN sampler on the `small` and `big`
models at 64 warmup / 64 samples (samples, probs, obs, potential, grad, step size, acceptance, diag and trace throughout);
and the edge paths of both samplers' outputs and of the fit: evaluate-only calls (W = S = 0) at an init whose potential is
finite for some chains and not for others, warmup-only calls (S = 0), chains started at a non-finite init with W + S > 0,
and the fit with max_iter = 0.
`compare` exits non-zero unless every tensor is bitwise equal (NaNs in the same places count as equal).
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIT_SHAPES = [(32, 40, 1), (16, 64, 3), (8, 128, 5), (100, 50, 1)]  # B, T, F; every prefix 1..T
# B, T, F, prefix step, warmup, samples, max tree depth, n_pred
GP_MCMC = [(100, 50, 1, 1, 300, 100, 10, 1), (100, 128, 5, 10, 300, 100, 10, 3), (32, 40, 2, 3, 100, 50, 2, 1)]
BNN_MODELS = [("small", 3, 5), ("big", 8, 64)]                      # name, F, E; 100 datasets, 100 training rows
BNN_STEPS = 64
# name, samples, warmup, whether every third chain starts at NaN and the others at 0 (otherwise the uniform draws)
EDGE_PATHS = [("evaluate_only", 0, 0, True), ("warmup_only", 0, 50, False), ("nonfinite_init", 20, 20, True)]


def run(out, tree):
    sys.path.insert(0, os.path.abspath(tree))
    import torch
    from transformerscandobayesianinference_b200 import mcmc_svi_transformer_on_bayesian as M
    from transformerscandobayesianinference_b200.priors import fast_gp_mix
    from transformerscandobayesianinference_b200.priors import pyro as P
    res = {}

    def keep(prefix, r):
        res.update({f"{prefix}/{n}": v.cpu() for n, v in r.items() if torch.is_tensor(v)})

    for k, (B, T, F) in enumerate(FIT_SHAPES):
        torch.manual_seed(100 + k)
        x, y, _ = fast_gp_mix.get_batch(B, T, F, device="cuda", batch_size_per_gp_sample=4 if B % 4 == 0 else 1)
        xb, yb = x.transpose(0, 1).contiguous(), y.transpose(0, 1).contiguous()
        keep(f"fit/{B}x{T}x{F}", fast_gp_mix.fit_map(xb, yb, list(range(1, T + 1)), {}, grad=True))
    for k, (B, T, F, step, W, S, depth, n_pred) in enumerate(GP_MCMC):
        torch.manual_seed(200 + k)
        x, y, _ = fast_gp_mix.get_batch(B, T, F, device="cuda", batch_size_per_gp_sample=4)
        xb, yb = x.transpose(0, 1).contiguous(), y.transpose(0, 1).contiguous()
        r = fast_gp_mix.sample_posterior(xb, yb, list(range(1, T, step)), {}, S, W, seed=1, max_tree_depth=depth,
                                         trace=True, n_pred=n_pred)
        keep(f"gp_mcmc/{B}x{T}x{F}/step{step}/depth{depth}", r)
    for name, F, E in BNN_MODELS:
        x, y = P.sample_bnn_prior(100, 300, F, E, "cuda", seed=7)
        X, Y = x.transpose(0, 1).contiguous(), y.transpose(0, 1).contiguous()
        spec = {"num_features": F, "embed": E}
        r = M.sample_bnn_posterior(X[:, :100], Y[:, :100], X[:, 100:], spec, BNN_STEPS, BNN_STEPS, seed=1, trace=True)
        keep(f"bnn_mcmc/{name}", r)

    def mixed_init(n, d):
        init = torch.zeros(n, d, dtype=torch.float64)
        init[::3] = float("nan")
        return init

    torch.manual_seed(300)
    B, T, F = FIT_SHAPES[0]
    x, y, _ = fast_gp_mix.get_batch(B, T, F, device="cuda", batch_size_per_gp_sample=4)
    xb, yb = x.transpose(0, 1).contiguous(), y.transpose(0, 1).contiguous()
    keep(f"fit/{B}x{T}x{F}/max_iter0", fast_gp_mix.fit_map(xb, yb, list(range(1, T + 1)), {}, max_iter=0, grad=True))
    ts = [5, 20, T]                                                    # t = T: no predictive row
    for name, S, W, nan_init in EDGE_PATHS:
        init = mixed_init(len(ts) * B, F + 2).view(len(ts), B, F + 2) if nan_init else None
        keep(f"gp_mcmc/{name}", fast_gp_mix.sample_posterior(xb, yb, ts, {}, S, W, seed=2, init=init, trace=True,
                                                             n_pred=2))
    x, y = P.sample_bnn_prior(30, 150, 3, 5, "cuda", seed=8)
    X, Y = x.transpose(0, 1).contiguous(), y.transpose(0, 1).contiguous()
    for name, S, W, nan_init in EDGE_PATHS:
        init = mixed_init(30, 3 * 5 + 3 * 5 + 2) if nan_init else None
        keep(f"bnn_mcmc/{name}", M.sample_bnn_posterior(X[:, :100], Y[:, :100], X[:, 100:], {"num_features": 3, "embed": 5},
                                                         S, W, seed=2, init=init, trace=True))
    torch.save(res, out)
    print(f"saved {len(res)} tensors from {tree} to {out}")


def compare(a_path, b_path):
    import torch
    a, b = torch.load(a_path), torch.load(b_path)
    if set(a) != set(b):
        raise SystemExit(f"different outputs: {sorted(set(a) ^ set(b))}")
    diff = [k for k in sorted(a) if not (a[k].shape == b[k].shape and torch.equal(a[k].isnan(), b[k].isnan())
                                         and torch.equal(a[k].nan_to_num(0.0), b[k].nan_to_num(0.0)))]
    print(f"{len(a)} tensors compared, {len(diff)} differ: {diff}")
    if diff:
        raise SystemExit(1)


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    r = sub.add_parser("run")
    r.add_argument("out")
    r.add_argument("--tree", default=ROOT)
    c = sub.add_parser("compare")
    c.add_argument("a")
    c.add_argument("b")
    args = ap.parse_args()
    if args.cmd == "run":
        run(args.out, args.tree)
    else:
        compare(args.a, args.b)


if __name__ == "__main__":
    main()
