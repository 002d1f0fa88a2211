"""Time encoders.Conv (forward + backward) with CUDA events at BASELINE configuration 5's shape (1536 images of 28 x 28)
and at the FewShotOmniglot notebook's 5-shot shape (T = 26 x B = 100), with the achieved TFLOP/s and the share of the
larger of the two lower bounds (tensor-core FLOPs at 989 TFLOP/s, activation bytes at 3.35 TB/s); the same stack in torch
bf16 channels-last (cuDNN) as a yardstick; and configuration 5's training-step throughput through build_trainer /
Trainer.step with the Omniglot sampler on a synthetic bank.  Prints the GPU name and power limit with the numbers.

    python tools/time_conv_encoder.py [--iters 50] [--profile]

--profile instead lists the kernels of five configuration-5 encoder steps by CUDA time (torch.profiler, a run of its own).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

from gpu_timing import card, event_times, kernel_seconds  # noqa: E402

PEAK_BF16, PEAK_BW = 989e12, 3.35e12      # H100 SXM data sheet (dense bf16, HBM3)


def stack_sides(S):
    sides, s = [], S
    while len(sides) < 5 and s >= 4:
        sides.append(s)
        s -= 2
    return sides


def flops(N, S, E):
    """Forward + backward FLOPs: every conv's forward and weight gradient, the data gradient of the 64 -> 64 convs (the
    input conv has none), the projection's three GEMMs."""
    f = 0.0
    for i, s in enumerate(stack_sides(S)):
        conv = 2.0 * N * (s - 2) ** 2 * 64 * 9 * (1 if i == 0 else 64)
        f += conv * (2 if i == 0 else 3)
    return f + 3 * 2.0 * N * 64 * E


def act_bytes(N, S, dt_size=2):
    """Activation traffic the stack cannot avoid: each conv's output is written and read by the next layer in the forward,
    read again as the ReLU mask and as the weight-gradient operand in the backward, and its gradient is written once and
    read twice (weight and data gradient); the images are read twice (forward, input-conv weight gradient)."""
    b = 2.0 * N * S * S * 4
    for s in stack_sides(S):
        b += 6.0 * N * (s - 2) ** 2 * 64 * dt_size
    return b


def time_ms(fn, iters):
    return 1e3 * event_times(fn, 1, warmup=5, calls=iters)[0]


def time_encoder(T, B, S, E, iters):
    from transformerscandobayesianinference_b200 import encoders
    torch.manual_seed(0)
    enc = encoders.Conv(S * S, E).cuda()
    x = torch.rand(T, B, S * S, device="cuda")
    dout = torch.randn(T, B, E, device="cuda")

    def ours():
        enc(x).backward(dout)

    # yardstick: the same stack in torch bf16 channels-last
    ref = nn.ModuleList([nn.Conv2d(1 if i == 0 else 64, 64, 3) for i in range(enc.n_conv)]).cuda().to(torch.bfloat16)
    ref = ref.to(memory_format=torch.channels_last)
    lin = nn.Linear(64, E).cuda().to(torch.bfloat16)
    xi = x.reshape(-1, 1, S, S).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    dref = dout.reshape(-1, E).to(torch.bfloat16)

    def cudnn():
        h = xi
        for c in ref:
            h = torch.relu(c(h))
        lin(h.mean((2, 3))).backward(dref)

    N = T * B
    f, by = flops(N, S, E), act_bytes(N, S)
    t_flop, t_byte = f / PEAK_BF16, by / PEAK_BW
    ms = time_ms(ours, iters)
    ms_ref = time_ms(cudnn, iters)
    bound = max(t_flop, t_byte)
    return {"shape": f"T={T} B={B} S={S} E={E}", "images": N, "ms": round(ms, 4), "tflops": round(f / ms / 1e9, 1),
            "gflop": round(f / 1e9, 1), "gbytes": round(by / 1e9, 3), "bound_ms": round(bound * 1e3, 4),
            "bound": "compute" if t_flop >= t_byte else "memory", "share_of_bound": round(bound * 1e3 / ms, 3),
            "cudnn_bf16_ms": round(ms_ref, 4)}


def time_cfg5_step(iters, E=512, B=256):
    import numpy as np
    from torch import nn as tnn
    from transformerscandobayesianinference_b200 import encoders, train
    from transformerscandobayesianinference_b200.priors import omniglot
    rng = np.random.default_rng(0)
    ink = (rng.random((1623, 1, 28, 28)) < 0.15) ^ (rng.random((1623, 20, 28, 28)) < 0.03)
    bank = omniglot.Bank(np.where(ink, 0, 255).astype(np.uint8), [("background", 0, 964), ("evaluation", 964, 659)])
    # the DataLoader reads its bank through `load_bank` (the extracted image tree under ./omniglot); serve the synthetic
    # bank instead, whatever the working directory
    omniglot.load_bank = lambda S, root='omniglot': bank
    tr = train.build_trainer(omniglot.DataLoader, tnn.CrossEntropyLoss(reduction='none'), encoders.Conv, emsize=E,
                             nhid=1024, nlayers=4, nhead=4, dropout=0.0, epochs=1, steps_per_epoch=iters, batch_size=B,
                             bptt=6, lr=1e-4, warmup_epochs=0, y_encoder_generator=encoders.get_Canonical(5),
                             extra_prior_kwargs_dict=dict(num_features=784, num_outputs=5), single_eval_pos_gen=5)
    batches = [next(iter(tr.dl)) for _ in range(4)]

    def step(i=[0]):
        (x, y), t = batches[i[0] % 4]
        i[0] += 1
        tr.step((x, y), t, 5)
    ms = time_ms(step, iters)
    return {"shape": f"cfg5 T=6 B={B} E={E} nhid=1024 4 layers", "step_ms": round(ms, 3),
            "sequences_per_s": round(B / ms * 1e3, 1)}


def profile_encoder(T=6, B=256, S=28, E=512):
    from transformerscandobayesianinference_b200 import encoders
    enc = encoders.Conv(S * S, E).cuda()
    x = torch.rand(T, B, S * S, device="cuda")
    dout = torch.randn(T, B, E, device="cuda")
    for _ in range(3):
        enc(x).backward(dout)
    kernels = kernel_seconds(lambda: [enc(x).backward(dout) for _ in range(5)])
    print(f"{'kernel':90s} {'total ms':>9s} {'launches':>8s} {'ms each':>8s}")
    for name, (s, n) in sorted(kernels.items(), key=lambda kv: -kv[1][0])[:20]:
        print(f"{name[:90]:90s} {s * 1e3:9.3f} {n:8d} {s / n * 1e3:8.3f}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    print(json.dumps({"gpu": card("time_conv_encoder")}))
    if args.profile:
        profile_encoder()
        return
    print(json.dumps(time_encoder(6, 256, 28, 512, args.iters)))
    print(json.dumps(time_encoder(26, 100, 28, 512, args.iters)))
    print(json.dumps(time_cfg5_step(args.iters)))


if __name__ == "__main__":
    main()
