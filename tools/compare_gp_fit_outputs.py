"""Checks that two builds of the library give bitwise equal MAP-fit results (`priors.fast_gp_mix.fit_map`).

Used when csrc/gp_fit.cu or csrc/gp_posterior.cuh change without meaning to change the fit, e.g. to compare the tree
against its parent commit on a GPU:

    git worktree add /tmp/parent HEAD~1 && (cd /tmp/parent && python -m transformerscandobayesianinference_b200.csrc.build)
    python tools/compare_gp_fit_outputs.py run /tmp/old.pt --tree /tmp/parent
    python tools/compare_gp_fit_outputs.py run /tmp/new.pt
    python tools/compare_gp_fit_outputs.py compare /tmp/old.pt /tmp/new.pt

`run` imports the package (and its library) from --tree (default: this checkout) and saves every output of seeded
fit_map calls at four shapes: theta, f, grad, mean, var, iters, nevals and status.  `compare` exits non-zero unless
every tensor is bitwise equal (NaNs in the same places count as equal).
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(32, 40, 1), (16, 64, 3), (8, 128, 5), (100, 50, 1)]      # B, T, F; every prefix 1..T


def run(out, tree):
    sys.path.insert(0, os.path.abspath(tree))
    import torch
    from transformerscandobayesianinference_b200.priors import fast_gp_mix
    res = {}
    for k, (B, T, F) in enumerate(SHAPES):
        torch.manual_seed(100 + k)
        x, y, _ = fast_gp_mix.get_batch(B, T, F, device="cuda", batch_size_per_gp_sample=4 if B % 4 == 0 else 1)
        xb, yb = x.transpose(0, 1).contiguous(), y.transpose(0, 1).contiguous()
        r = fast_gp_mix.fit_map(xb, yb, list(range(1, T + 1)), {}, grad=True)
        res.update({f"{B}x{T}x{F}/{n}": v.cpu() for n, v in r.items()})
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
