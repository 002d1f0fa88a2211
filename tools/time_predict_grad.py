"""Time the gradient of `predict` with respect to the query points, on the GP-regression model of the reference's
GP-fitting experiments (emsize 512, 4 heads, 6 layers, nhid 1024, 1000 buckets), at n training rows and m query rows per
dataset, B datasets:

  1. `predict` alone (no graph) against `predict` with a graph plus its backward to x_query;
  2. the context-attention backward kernel alone, with its bytes and FLOPs from the shapes and its share of the larger of
     the two H100 bounds.

    python tools/time_predict_grad.py [--n 1000] [--m 10000] [--B 1 16] [--reps 5]
"""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.gpu_timing import card, event_times  # noqa: E402
from transformerscandobayesianinference_b200 import _lib_input_grad as LIG, encoders, engine, transformer  # noqa: E402

E, H, NL, NHID, N_OUT, F = 512, 4, 6, 1024, 1000, 1
PEAK_BF16, PEAK_FP32, PEAK_BYTES = 989e12, 67e12, 3.35e12     # H100 SXM data sheet (dense), 700 W


def _model():
    torch.manual_seed(0)
    m = transformer.TransformerModel(encoders.Linear(F, E), N_OUT, E, H, NHID, NL, 0.0, y_encoder=encoders.Linear(1, E))
    with torch.no_grad():
        for layer in m.transformer_encoder.layers:
            layer.linear2.weight.normal_(0, 0.02)
            layer.self_attn.out_proj.weight.normal_(0, 0.02)
    return m.cuda().eval()


def backward_work(m, n, B, dtype_bytes):
    """(FLOPs, bytes) the context backward needs: S = q K^T, dP = dO V^T and dQ += dS K over the n cached keys per (row,
    head), plus the own key's dot products; Q | K | V and dO of the query rows, the cache, O (delta) read once, and
    dQ | dK | dV written once."""
    dh = E // H
    flops = 6.0 * m * B * H * n * dh + 6.0 * m * B * H * dh
    nbytes = dtype_bytes * (3 * m * B * E + m * B * E + 2 * n * B * E + m * B * E + 3 * m * B * E)
    return flops, nbytes


def run(n, m, B, reps):
    model = _model()
    g = torch.Generator(device="cuda").manual_seed(n + m + B)
    x_tr, y_tr = torch.rand(n, B, F, device="cuda", generator=g), torch.randn(n, B, device="cuda", generator=g)
    x_q = torch.rand(m, B, F, device="cuda", generator=g)
    with torch.no_grad():
        ctx = model.encode_context(x_tr, y_tr)

    def plain():
        with torch.no_grad():
            model.predict(ctx, x_q)

    def with_grad():
        xq = x_q.clone().requires_grad_(True)
        model.predict(ctx, xq).sum().backward()

    t_plain = event_times(plain, reps)[reps // 2]
    t_grad = event_times(with_grad, reps)[reps // 2]

    dt = engine.act_dtype(model.precision)
    dh = E // H
    qkv = torch.randn(m * B, 3 * E, device="cuda").to(dt)
    dout = torch.randn(m * B, E, device="cuda").to(dt)
    out = torch.empty(m * B, E, device="cuda", dtype=dt)
    lse = torch.empty(B * H, m, device="cuda")
    LIG.attention_ctx_grad_fwd(qkv, ctx.kv[0], out, lse, m, n, B, H, dh)
    dqkv = torch.empty_like(qkv)
    delta = torch.empty_like(lse)
    t_k = event_times(lambda: LIG.attention_ctx_bwd(qkv, ctx.kv[0], out, lse, dout, dqkv, delta, m, n, B, H, dh), reps,
                      warmup=3, calls=20)[reps // 2]
    flops, nbytes = backward_work(m, n, B, 2 if dt == torch.bfloat16 else 4)
    t_flops = flops / (PEAK_BF16 if dt == torch.bfloat16 else PEAK_FP32)
    t_bytes = nbytes / PEAK_BYTES
    bound = "compute" if t_flops >= t_bytes else "memory"
    print(f"n = {n}, m = {m}, B = {B}:")
    print(f"  predict alone            {t_plain * 1e3:10.3f} ms")
    print(f"  predict + backward       {t_grad * 1e3:10.3f} ms  ({t_grad / t_plain:.2f} x)")
    print(f"  context backward kernel  {t_k * 1e6:10.1f} us  ({flops / 1e9:.2f} GFLOP, {nbytes / 1e6:.1f} MB; "
          f"{flops / t_k / 1e12:.1f} TFLOP/s, {nbytes / t_k / 1e9:.0f} GB/s; {bound}-bound: "
          f"{max(t_flops, t_bytes) / t_k * 100:.1f} % of that bound)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000)
    ap.add_argument("--m", type=int, default=10_000)
    ap.add_argument("--B", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    print(card("time_predict_grad"))
    print(f"precision {engine.default_precision()}; E {E}, {H} heads, {NL} layers, nhid {NHID}, {N_OUT} buckets; "
          f"median of each sample set")
    for B in args.B:
        run(args.n, args.m, B, args.reps)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"({time.time() - t0:.0f} s)")
