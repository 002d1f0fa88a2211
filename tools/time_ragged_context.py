"""Time training sets of different sizes in one batch (`encode_context(x_train, y_train, n_train)` + one `predict`)
against a loop over the sizes (one uniform `encode_context` + `predict` per size), at two shapes:

  bnn      the Bayesian-NN experiment: emsize 256, 4 heads, 5 layers, nhid 512, 8 features; D datasets each scored at
           the 19 training-set sizes 2, 7, .., 92 (a ragged batch of 19 D datasets); 208 query rows per dataset
  tabular  the tabular evaluation: emsize 512, 4 heads, 6 layers, nhid 1024, 100 features; D datasets each scored at the
           eval positions 10, 20, 40; 200 query rows per dataset

and the uniform path alone (n_train=None, every dataset at the largest size), so that the same script run on two
builds shows what the ragged support costs a caller who does not use it (`--uniform-only` times just that).

    python tools/time_ragged_context.py [--datasets 64] [--reps 7] [--uniform-only]
"""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.gpu_timing import card, event_times  # noqa: E402
from transformerscandobayesianinference_b200 import encoders, engine, transformer  # noqa: E402

BNN_SIZES = list(range(2, 93, 5))
SHAPES = {
    "bnn": dict(E=256, H=4, NL=5, NHID=512, F=8, N_OUT=1, sizes=BNN_SIZES, m=208),
    "tabular": dict(E=512, H=4, NL=6, NHID=1024, F=100, N_OUT=1, sizes=[10, 20, 40], m=200),
}


def _model(s):
    torch.manual_seed(0)
    m = transformer.TransformerModel(encoders.Linear(s["F"], s["E"]), s["N_OUT"], s["E"], s["H"], s["NHID"], s["NL"], 0.0,
                                     y_encoder=encoders.Linear(1, s["E"]))
    with torch.no_grad():
        for layer in m.transformer_encoder.layers:
            layer.linear2.weight.normal_(0, 0.02)
            layer.self_attn.out_proj.weight.normal_(0, 0.02)
    return m.cuda().eval()


def run(name, s, D, reps, uniform_only):
    model = _model(s)
    sizes, n, m = s["sizes"], max(s["sizes"]), s["m"]
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(n + m, D, s["F"], device="cuda", generator=g)
    y = (torch.rand(n + m, D, device="cuda", generator=g) > 0.5).float()
    k = len(sizes)
    # the ragged batch: dataset d at size sizes[j] is column j * D + d
    xr, yr, xq = x[:n].repeat(1, k, 1), y[:n].repeat(1, k), x[n:].repeat(1, k, 1)
    n_train = torch.tensor([v for v in sizes for _ in range(D)], device="cuda")
    med = lambda ts: ts[len(ts) // 2]
    out = {}
    with torch.no_grad():
        out["uniform n_max"] = med(event_times(lambda: model.predict(model.encode_context(xr, yr), xq), reps, warmup=2))
        if not uniform_only:
            loop = lambda: [model.predict(model.encode_context(x[:v], y[:v]), x[n:]) for v in sizes]
            out["per-size loop"] = med(event_times(loop, reps, warmup=2))
            out["one ragged call"] = med(event_times(lambda: model.predict(model.encode_context(xr, yr, n_train), xq), reps,
                                                     warmup=2))
            ragged = model.predict(model.encode_context(xr, yr, n_train), xq)
            alone = torch.cat([model.predict(model.encode_context(x[:v], y[:v]), x[n:]) for v in sizes], 1)
            same = torch.equal(ragged, alone)
    print(f"{name}: E {s['E']}, {s['H']} heads, {s['NL']} layers, nhid {s['NHID']}, F {s['F']}; {D} datasets x "
          f"{k} sizes {sizes[0]}..{n}; {m} query rows; precision {model.precision}")
    for key, t in out.items():
        print(f"  {key:16s} {t * 1e3:9.3f} ms")
    if not uniform_only:
        print(f"  speed-up of one ragged call over the loop: {out['per-size loop'] / out['one ragged call']:.2f} x; "
              f"ragged == per-size results bitwise: {same}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--datasets", type=int, default=64)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--uniform-only", action="store_true")
    args = ap.parse_args()
    print(card("time_ragged_context"))
    print(f"default precision {engine.default_precision()}; median of {args.reps} samples, each one CUDA-event bracket")
    for name, s in SHAPES.items():
        run(name, s, args.datasets, args.reps, args.uniform_only)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"({time.time() - t0:.0f} s)")
