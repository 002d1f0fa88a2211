"""Time inference against a cached training set (`TransformerModel.encode_context` + `predict`) against the full
`forward` on the concatenated sequence, on the GP-regression model of the reference's GP-fitting experiments (emsize 512,
4 heads, 6 layers, nhid 1024, a 1000-bucket FullSupportBarDistribution head), B = 16 datasets, for n training rows:

  1. one query set of 10 000 rows: one forward against encode_context + one predict;
  2. 100 query sets of 1 000 rows: 100 forward calls against one encode_context + 100 predict calls;
  3. the context-attention kernel alone (10 000 query rows), with its bytes and FLOPs from the shapes and its share of
     the larger of the two H100 bounds.

    python tools/time_context_inference.py [--n 100 1000 2000] [--reps 5]
"""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.gpu_timing import card, event_times  # noqa: E402
from transformerscandobayesianinference_b200 import _lib as L, encoders, engine, transformer  # noqa: E402

E, H, NL, NHID, N_OUT, F, B = 512, 4, 6, 1024, 1000, 1, 16
M_ONE, M_SET, N_SETS = 10_000, 1_000, 100
PEAK_BF16, PEAK_FP32, PEAK_BYTES = 989e12, 67e12, 3.35e12     # H100 SXM data sheet (dense), 700 W


def _model():
    torch.manual_seed(0)
    m = transformer.TransformerModel(encoders.Linear(F, E), N_OUT, E, H, NHID, NL, 0.0, y_encoder=encoders.Linear(1, E))
    with torch.no_grad():
        for layer in m.transformer_encoder.layers:
            layer.linear2.weight.normal_(0, 0.02)
            layer.self_attn.out_proj.weight.normal_(0, 0.02)
    return m.cuda().eval()


def attention_work(m, n, dtype_bytes):
    """(FLOPs, bytes) the context attention needs: S = q K^T and O = P V over n + 1 keys per (row, head); Q, the query
    rows' own K and V, the cache and O each moved once."""
    dh = E // H
    flops = 4.0 * m * B * H * (n + 1) * dh
    nbytes = dtype_bytes * (3 * m * B * E + 2 * n * B * E + m * B * E)
    return flops, nbytes


def run(n, reps):
    model = _model()
    g = torch.Generator(device="cuda").manual_seed(n)
    x_tr, y_tr = torch.rand(n, B, F, device="cuda", generator=g), torch.randn(n, B, device="cuda", generator=g)
    x_one = torch.rand(M_ONE, B, F, device="cuda", generator=g)
    x_sets = torch.rand(N_SETS, M_SET, B, F, device="cuda", generator=g)
    y_pad = torch.zeros(M_ONE, B, device="cuda")
    fwd = lambda xq: model((torch.cat([x_tr, xq], 0), torch.cat([y_tr, y_pad[:xq.shape[0]]], 0)), single_eval_pos=n)
    out = {}
    with torch.no_grad():
        ctx = model.encode_context(x_tr, y_tr)
        diff = (model.predict(ctx, x_one) - fwd(x_one)).abs().max().item()
        out["one forward"] = event_times(lambda: fwd(x_one), reps)[reps // 2]
        out["one encode+predict"] = event_times(lambda: model.predict(model.encode_context(x_tr, y_tr), x_one), reps)[reps // 2]
        out["100 forward"] = event_times(lambda: [fwd(xq) for xq in x_sets], max(reps // 2, 1))[max(reps // 2, 1) // 2]

        def sets():
            c = model.encode_context(x_tr, y_tr)
            for xq in x_sets:
                model.predict(c, xq)
        out["1 encode+100 predict"] = event_times(sets, max(reps // 2, 1))[max(reps // 2, 1) // 2]

        dt = engine.act_dtype(model.precision)
        qkv = torch.randn(M_ONE * B, 3 * E, device="cuda").to(dt)
        att = torch.empty(M_ONE * B, E, device="cuda", dtype=dt)
        kv = ctx.kv[0]
        t_k = event_times(lambda: L.attention_ctx_fwd(qkv, kv, att, M_ONE, n, B, H, E // H), reps, warmup=3,
                          calls=20)[reps // 2]
    flops, nbytes = attention_work(M_ONE, n, 2 if dt == torch.bfloat16 else 4)
    t_flops = flops / (PEAK_BF16 if dt == torch.bfloat16 else PEAK_FP32)
    t_bytes = nbytes / PEAK_BYTES
    bound = "compute" if t_flops >= t_bytes else "memory"
    print(f"n = {n}: max |predict - forward| over the 10 000-row set = {diff:.3g}")
    for name, s in out.items():
        print(f"  {name:22s} {s * 1e3:10.3f} ms")
    print(f"  speed-up, one set      {out['one forward'] / out['one encode+predict']:10.2f} x")
    print(f"  speed-up, 100 sets     {out['100 forward'] / out['1 encode+100 predict']:10.2f} x")
    print(f"  context attention      {t_k * 1e6:10.1f} us  ({flops / 1e9:.2f} GFLOP, {nbytes / 1e6:.1f} MB; "
          f"{flops / t_k / 1e12:.1f} TFLOP/s, {nbytes / t_k / 1e9:.0f} GB/s; {bound}-bound: "
          f"{max(t_flops, t_bytes) / t_k * 100:.1f} % of that bound)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[100, 1000, 2000])
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    print(card("time_context_inference"))
    print(f"precision {engine.default_precision()}; E {E}, {H} heads, {NL} layers, nhid {NHID}, {N_OUT} buckets, B {B}; "
          f"median of each sample set")
    for n in args.n:
        run(n, args.reps)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"({time.time() - t0:.0f} s)")
