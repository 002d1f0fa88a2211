"""Per-kernel-family time breakdown of one cfg-2 training step (CUDA events around every C-ABI call).

Debug/measurement aid: wraps the ctypes entry points of libpfn_b200.so with event timing, runs a few steps, prints the
time per entry point (GEMMs grouped by shape/epilogue/operand layout) and the remainder (torch-side elementwise, Adam, ...).
Each wrapped call is timed on its own, synchronised before and after, so every row includes one launch latency and the
sum is an upper bound of the kernels' own time; the step time comes from a separate window of steps without them.

For every wgmma GEMM row it also prints the algorithmic HBM bytes (operands, aux, C and C2 once each: _lib.gemm_bytes,
the formula of _lib.PROFILE_GEMM), the achieved TFLOP/s and GB/s, and the share of the floor, floor = max(FLOP / peak,
bytes / bandwidth) with the H100 SXM data-sheet peaks (dense BF16 989 TFLOP/s, HBM3 3.35 TB/s); the bound that sets the
floor is named.  Tensor-core attention rows print their algorithmic FLOPs (mask-aware) and the achieved TFLOP/s."""
import sys, os, collections
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from transformerscandobayesianinference_b200 import _lib as L, priors, bar_distribution, transformer, encoders
from gpu_timing import attention_pairs, card, event_times

T, F, E, NL, NH, H, NB, sep = 1000, 1, 512, 6, 1024, 4, 100, 500
PEAK_FLOPS, PEAK_BW = 989e12, 3.35e12
REC = None          # while a list: (label, seconds) of every wrapped call is appended to it
GEMM_COST = {}      # label -> (flop, bytes) of one call
ATTN_COST = {}      # label -> algorithmic flop of one call
NAMES = ["pfn_gemm_bf16_tc", "pfn_gemm_simt", "pfn_attention_fwd_tc", "pfn_attention_bwd_tc", "pfn_attention_fwd_simt",
         "pfn_attention_bwd_simt", "pfn_embed_fwd", "pfn_embed_bwd", "pfn_layernorm_fwd", "pfn_layernorm_bwd", "pfn_colsum",
         "pfn_bar_nll_fwd", "pfn_bar_nll_bwd", "pfn_gp_sample"]


def wrap(lib, name):
    orig = getattr(lib, name)
    def f(*a):
        if REC is None:
            return orig(*a)
        label = name
        if name.startswith("pfn_gemm"):
            d = a[0]._obj
            label = f"gemm M={d.M} N={d.N} K={d.K} epi={d.epilogue} amn={d.a_mn_major} bmn={d.b_mn_major} c2={int(bool(d.C2))} aux={int(bool(d.aux))} cdt={d.c_dtype} ks={d.k_splits}"
            if name == "pfn_gemm_bf16_tc":
                GEMM_COST[label] = (2.0 * d.M * d.N * d.K, L.gemm_bytes(d))
        elif name in ("pfn_attention_fwd_tc", "pfn_attention_bwd_tc"):
            # matmul passes over the attended (query, key) pairs: forward S and PV (2 passes), backward S, dP, dV, dK, dQ
            # (5 passes; recomputed S / dP not counted)
            d = a[0]._obj
            label = f"{name} T={d.T} B={d.B} H={d.H} sep={d.sep}"
            ATTN_COST[label] = (2 if name.endswith("fwd_tc") else 5) * 2.0 * attention_pairs(d.T, d.sep) * d.dh * d.B * d.H
        rc = []
        REC.append((label, event_times(lambda: rc.append(orig(*a)), 1, warmup=0)[0]))
        return rc[0]
    setattr(lib, name, f)


def main():
    global REC
    dev = torch.device("cuda:0")
    B = int(os.environ.get("PFN_BENCH_B", 512))
    print(f"card: {card('step_breakdown')}")
    lib = L.load()
    for n in NAMES:
        wrap(lib, n)

    enc = encoders.Linear(F, E)
    yenc = encoders.Linear(1, E)
    model = transformer.TransformerModel(enc, NB, E, H, NH, NL, 0.0, y_encoder=yenc, input_normalization=False).to(dev)
    ys = priors.fast_gp.get_batch(64, T, F, device=str(dev), hyperparameters={"noise": 1e-4, "outputscale": 1., "lengthscale": .6})[1]
    crit = bar_distribution.FullSupportBarDistribution(bar_distribution.get_bucket_limits(NB, ys=ys.float().cpu())).to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=1e-4, fused=True)
    ls = torch.full((B, F), .6, device=dev); os_ = torch.ones(B, device=dev); nz = torch.full((B,), 1e-4, device=dev)
    bar_distribution.BarDistribution.defer_support_check = True

    def step():
        x_bt = torch.rand(B, T, F, device=dev); z_bt = torch.randn(B, T, device=dev)
        y_bt = priors.fast_gp.sample_gp(x_bt, z_bt, ls, os_, nz)
        x, y = x_bt.transpose(0, 1), y_bt.transpose(0, 1)
        logits = model((x, y), single_eval_pos=sep)
        loss = crit(logits.reshape(-1, NB), y[sep:].flatten()).mean()
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 1.)
        opt.step(); opt.zero_grad(set_to_none=True)

    NS = 3
    total = 1e3 * event_times(step, 1, warmup=3, calls=NS)[0]
    REC = []
    for _ in range(NS): step()
    agg = collections.OrderedDict()
    for label, sec in REC:
        c = agg.setdefault(label, [0, 0.0]); c[0] += 1; c[1] += 1e3 * sec
    rows = sorted(agg.items(), key=lambda kv: -kv[1][1])
    s = 0.0
    print(f"step {total:.2f} ms")
    for label, (n, t) in rows:
        extra = ""
        if label in GEMM_COST:
            flop, nbytes = GEMM_COST[label]
            sec = t / n * 1e-3
            t_flop, t_bytes = flop / PEAK_FLOPS, nbytes / PEAK_BW
            extra = (f"  | {nbytes / 1e9:6.3f} GB {flop / sec / 1e12:6.1f} TFLOP/s {nbytes / sec / 1e9:7.1f} GB/s"
                     f"  floor {max(t_flop, t_bytes) * 1e3:6.3f} ms ({'tensor' if t_flop >= t_bytes else 'HBM'})"
                     f"  {100 * max(t_flop, t_bytes) / sec:5.1f}% of floor")
        if label in ATTN_COST:
            extra = f"  | {ATTN_COST[label] / 1e9:8.1f} GFLOP {ATTN_COST[label] / (t / n * 1e-3) / 1e12:6.1f} TFLOP/s"
        print(f"{t / NS:8.3f} ms/step  {n // NS:3d}x  {t / n:7.3f} ms each  {label}{extra}")
        s += t / NS
    print(f"{s:8.3f} ms/step in C-ABI kernels; {total - s:.3f} ms/step elsewhere (torch elementwise, Adam, clip, launch gaps)")


if __name__ == "__main__":
    main()
