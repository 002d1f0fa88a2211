"""Time the tensor-core attention forward (pfn_attention_fwd_tc) and backward (pfn_attention_bwd_tc) of one or more builds of
libpfn_b200.so on the same inputs.

    python tools/time_attention.py [--profile] LIB [LIB ...]

Every library is loaded with ctypes and called with the same seeded qkv and dO at the cfg-2 shape (T = 1000, sep = 500,
B = 512, H = 4) and the cfg-4 shape (T = 2000, sep = 1000, B = 256, H = 4).  After a warm-up, each round times 30
launches per library with CUDA events, alternating the libraries, over 3 rounds.  It prints ms per launch and the
algorithmic TFLOP/s (the pair count of tools/step_breakdown.py: forward S and PV, backward S, dP, dV, dK and dQ over
T * sep + (T - sep) pairs).  The backward is called the way the engine calls it: out and lse from the first library's
forward, delta precomputed token-major ([T*B, H], delta_token_major = 1) and dq_colsum set.

Against the first library it prints the max and 99.9th-percentile |out - out_first| and the max |lse - lse_first|, and
for the backward the max |d dqkv| of dQ and of dK/dV, each split into rows < sep and rows >= sep, with the largest
difference in bf16 ulps of the first library's value, and the max |d dq_colsum|.

--profile also runs each library's backward under torch.profiler (in a pass of its own, after the timed rounds) and prints
the mean CUDA time of each of its kernels.  The card name, power limit and max SM clock are printed with the numbers."""
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
    for fn in (lib.pfn_attention_fwd_tc, lib.pfn_attention_bwd_tc):
        fn.restype = ctypes.c_int
        fn.argtypes = [ctypes.POINTER(L.AttnDesc), ctypes.c_void_p]
    return lib


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        q = f"{torch.cuda.get_device_name()}, power limit not read, max SM clock not read"
    return q


def time_rounds(launch, n):
    """ms per launch of launch(k) for each of n libraries, alternated over ROUNDS rounds after a warm-up"""
    for k in range(n):
        for _ in range(WARMUP):
            launch(k)
    torch.cuda.synchronize()
    times = [[] for _ in range(n)]
    for _ in range(ROUNDS):
        for k in range(n):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(LAUNCHES):
                launch(k)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / LAUNCHES)
    return times


def print_times(paths, times, flop):
    for k, p in enumerate(paths):
        ms = " / ".join(f"{t:.3f}" for t in times[k])
        print(f"  {p}: {ms} ms  ({flop / (min(times[k]) * 1e-3) / 1e12:.1f} TFLOP/s at the best round)")


def bf16_ulp(x):
    """spacing of bf16 numbers at |x| (8 significand bits)"""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def diff_line(name, a, ref):
    d = (a - ref).abs()
    if d.numel() == 0:
        return f"{name}: empty"
    ulps = (d / bf16_ulp(ref)).max().item()
    return f"{name}: max |d| {d.max().item():.3e} ({ulps:.2f} bf16 ulp), bit-identical {bool(torch.equal(a, ref))}"


def profile_bwd(paths, launch):
    from torch.profiler import ProfilerActivity, profile
    for k, p in enumerate(paths):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(LAUNCHES):
                launch(k)
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            if ev.device_type == torch.autograd.DeviceType.CUDA and ev.count > 0:
                us = getattr(ev, "device_time_total", None) or ev.cuda_time_total
                print(f"  profile {p}: {ev.key[:60]}: {us / ev.count / 1e3:.3f} ms x {ev.count}")


def main():
    args = sys.argv[1:]
    want_profile = "--profile" in args
    paths = [a for a in args if a != "--profile"]
    if not paths:
        sys.exit(__doc__)
    torch.cuda.init()
    libs = [open_lib(p) for p in paths]
    stream = torch.cuda.current_stream().cuda_stream
    print(f"card: {card()}")

    def call(k, fn, desc):
        rc = getattr(libs[k], fn)(ctypes.byref(desc), ctypes.c_void_p(stream))
        if rc != 0:
            raise RuntimeError(f"{paths[k]}: {libs[k].pfn_last_error().decode()}")

    for name, T, sep, B, H in SHAPES:
        E = H * DH
        g = torch.Generator(device="cuda").manual_seed(1234 + T)
        qkv = torch.randn(T * B, 3 * E, device="cuda", generator=g).to(torch.bfloat16)
        outs = [torch.empty(T * B, E, device="cuda", dtype=torch.bfloat16) for _ in libs]
        lses = [torch.empty(B * H, T, device="cuda") for _ in libs]
        descs = [L.attention_desc(qkv, o, s, T, B, H, DH, sep) for o, s in zip(outs, lses)]
        pairs = T * sep + (T - sep)

        times = time_rounds(lambda k: call(k, "pfn_attention_fwd_tc", descs[k]), len(libs))
        flop = 2 * 2.0 * pairs * DH * B * H
        print(f"{name} forward: T={T} sep={sep} B={B} H={H}, {flop / 1e9:.1f} GFLOP per launch")
        print_times(paths, times, flop)
        ref_o, ref_l = outs[0].float(), lses[0]
        for k in range(1, len(libs)):
            d = (outs[k].float() - ref_o).abs().flatten()
            n999 = max(1, d.numel() // 1000)
            p999 = d.topk(n999).values[-1].item()
            dl = (lses[k] - ref_l).abs().max().item()
            print(f"  {paths[k]} vs {paths[0]}: max |dout| {d.max().item():.3e}, 99.9th pct |dout| {p999:.3e} "
                  f"(max |out| {ref_o.abs().max().item():.3f}), max |dlse| {dl:.3e} (max |lse| {ref_l.abs().max().item():.3f})")

        # backward on the first library's forward outputs
        out, lse = outs[0], lses[0]
        del outs, lses, descs
        dout = (0.1 * torch.randn(T * B, E, device="cuda", generator=g)).to(torch.bfloat16)
        delta = (dout.float() * out.float()).view(T * B, H, DH).sum(-1).contiguous()    # token-major [T*B, H]
        dqkvs = [torch.empty(T * B, 3 * E, device="cuda", dtype=torch.bfloat16) for _ in libs]
        colsums = [torch.zeros(E, device="cuda") for _ in libs]
        bdescs = []
        for dq, cs in zip(dqkvs, colsums):
            d = L.attention_desc(qkv, out, lse, T, B, H, DH, sep, dout, dq, delta)
            d.dq_colsum, d.delta_token_major = cs.data_ptr(), 1
            bdescs.append(d)
        bwd = lambda k: call(k, "pfn_attention_bwd_tc", bdescs[k])
        times = time_rounds(bwd, len(libs))
        flop = 5 * 2.0 * pairs * DH * B * H
        print(f"{name} backward (token-major delta, dq_colsum): {flop / 1e9:.1f} GFLOP per launch")
        print_times(paths, times, flop)
        if want_profile:
            profile_bwd(paths, bwd)
        for k in range(len(libs)):
            dqkvs[k].zero_()
            colsums[k].zero_()
            bwd(k)
        torch.cuda.synchronize()
        ref = dqkvs[0].float().view(T, B, 3 * E)
        for k in range(1, len(libs)):
            a = dqkvs[k].float().view(T, B, 3 * E)
            print(f"  {paths[k]} vs {paths[0]}:")
            print("    " + diff_line("dQ rows < sep", a[:sep, :, :E], ref[:sep, :, :E]))
            print("    " + diff_line("dQ rows >= sep", a[sep:, :, :E], ref[sep:, :, :E]))
            print("    " + diff_line("dK/dV rows < sep", a[:sep, :, E:], ref[:sep, :, E:]))
            print("    " + diff_line("dK/dV rows >= sep", a[sep:, :, E:], ref[sep:, :, E:]))
            dc = (colsums[k] - colsums[0]).abs().max().item()
            print(f"    dq_colsum: max |d| {dc:.3e} (max |dq_colsum| {colsums[0].abs().max().item():.3f})")
        del qkv, out, lse, dout, delta, dqkvs, colsums, bdescs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
