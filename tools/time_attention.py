"""Time the tensor-core attention forward (pfn_attention_fwd_tc) of one or more builds of libpfn_b200.so on the same inputs.

    python tools/time_attention.py LIB [LIB ...]

Every library is loaded with ctypes and called with the same seeded qkv at the cfg-2 shape (T = 1000, sep = 500,
B = 512, H = 4) and the cfg-4 shape (T = 2000, sep = 1000, B = 256, H = 4).  After a warm-up, each round times 30
launches per library with CUDA events, alternating the libraries, over 3 rounds.  It prints ms per launch and the
algorithmic TFLOP/s (the pair count of tools/step_breakdown.py: S and PV over T * sep + (T - sep) pairs), then the max
and 99.9th-percentile |out - out_first| and the max |lse - lse_first| of each library against the first one.  The card
name, power limit and max SM clock are printed with the numbers."""
import ctypes
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from transformerscandobayesianinference_b200 import _lib as L

SHAPES = [("cfg2", 1000, 500, 512, 4), ("cfg4", 2000, 1000, 256, 4)]
DH, LAUNCHES, ROUNDS, WARMUP = 128, 30, 3, 3


def open_lib(path):
    lib = ctypes.CDLL(os.path.abspath(path))
    lib.pfn_last_error.restype = ctypes.c_char_p
    lib.pfn_attention_fwd_tc.restype = ctypes.c_int
    lib.pfn_attention_fwd_tc.argtypes = [ctypes.POINTER(L.AttnDesc), ctypes.c_void_p]
    return lib


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        q = f"{torch.cuda.get_device_name()}, power limit not read, max SM clock not read"
    return q


def main():
    paths = sys.argv[1:]
    if not paths:
        sys.exit(__doc__)
    torch.cuda.init()
    libs = [open_lib(p) for p in paths]
    stream = torch.cuda.current_stream().cuda_stream
    print(f"card: {card()}")
    for name, T, sep, B, H in SHAPES:
        E = H * DH
        g = torch.Generator(device="cuda").manual_seed(1234 + T)
        qkv = torch.randn(T * B, 3 * E, device="cuda", generator=g).to(torch.bfloat16)
        outs = [torch.empty(T * B, E, device="cuda", dtype=torch.bfloat16) for _ in libs]
        lses = [torch.empty(B * H, T, device="cuda") for _ in libs]
        descs = [L.attention_desc(qkv, o, s, T, B, H, DH, sep) for o, s in zip(outs, lses)]

        def launch(k):
            rc = libs[k].pfn_attention_fwd_tc(ctypes.byref(descs[k]), ctypes.c_void_p(stream))
            if rc != 0:
                raise RuntimeError(f"{paths[k]}: {libs[k].pfn_last_error().decode()}")

        for k in range(len(libs)):
            for _ in range(WARMUP):
                launch(k)
        torch.cuda.synchronize()
        times = [[] for _ in libs]
        for _ in range(ROUNDS):
            for k in range(len(libs)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(LAUNCHES):
                    launch(k)
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1) / LAUNCHES)
        flop = 2 * 2.0 * (T * sep + (T - sep)) * DH * B * H
        print(f"{name}: T={T} sep={sep} B={B} H={H}, {flop / 1e9:.1f} GFLOP per launch")
        for k, p in enumerate(paths):
            ms = " / ".join(f"{t:.3f}" for t in times[k])
            best = min(times[k])
            print(f"  {p}: {ms} ms  ({flop / (best * 1e-3) / 1e12:.1f} TFLOP/s at the best round)")
        ref_o, ref_l = outs[0].float(), lses[0]
        for k in range(1, len(libs)):
            d = (outs[k].float() - ref_o).abs().flatten()
            n999 = max(1, d.numel() // 1000)
            p999 = d.topk(n999).values[-1].item()
            dl = (lses[k] - ref_l).abs().max().item()
            print(f"  {paths[k]} vs {paths[0]}: max |dout| {d.max().item():.3e}, 99.9th pct |dout| {p999:.3e} "
                  f"(max |out| {ref_o.abs().max().item():.3f}), max |dlse| {dl:.3e} (max |lse| {ref_l.abs().max().item():.3f})")
        del qkv, outs, lses, descs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
