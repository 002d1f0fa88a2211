"""Time priors.stroke: the device sampler at the FewShotOmniglot notebook's batch (1000 datasets x 26 images of 28 x 28,
5 classes, last-index mode) and at B = 512 with CUDA events, its kernels with torch.profiler, the unmodified reference
sampler on the host cores (given a reference checkout, and when PIL imports), one Trainer.step at the notebook's model shape with a
pre-drawn batch against the step fed by the prefetching loader, and a short `train(priors.stroke.DataLoader, ...)` run
at the notebook's settings.

    python tools/time_stroke_prior.py [--iters 20] [--train-steps 10] [--reference-dir <reference checkout>]
"""
import argparse
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

T, C, F = 26, 5, 784
KW = dict(num_features=F, num_outputs=C, only_train_for_last_idx=True)


def time_device(stroke, B, iters):
    for _ in range(3):
        stroke.get_batch(B, T, device='cuda:0', **KW)
    torch.cuda.synchronize()
    ms = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        stroke.get_batch(B, T, device='cuda:0', **KW)
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return statistics.median(ms), min(ms)


def profile_kernels(stroke, B):
    from torch.profiler import profile, ProfilerActivity
    stroke.get_batch(B, T, device='cuda:0', **KW)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            stroke.get_batch(B, T, device='cuda:0', **KW)
        torch.cuda.synchronize()
    rows = []
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        if t > 0 and ev.count > 0:
            rows.append((t / ev.count, ev.count, ev.key))
    for us, n, key in sorted(rows, reverse=True)[:10]:
        print(f"    {us:9.1f} us  x{n:<3d} {key[:90]}")


def time_reference(B, reference_dir):
    try:
        import PIL  # noqa: F401
        import torchvision  # noqa: F401
    except ImportError as e:
        print(f"reference: {e}; skipped")
        return
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from make_stroke_golden import load_reference_stroke
    ref = load_reference_stroke(reference_dir)
    t0 = time.perf_counter()
    ref.get_batch(B, T, **KW)
    dt = time.perf_counter() - t0
    print(f"reference get_batch B={B}: {dt * 1e3:.0f} ms on the host (one Python thread; {os.cpu_count()} cores visible, "
          f"torch threads {torch.get_num_threads()})")


def time_steps(stroke, steps):
    from transformerscandobayesianinference_b200 import encoders
    from transformerscandobayesianinference_b200.train import Losses, build_trainer
    torch.manual_seed(0)
    tr = build_trainer(stroke.DataLoader, Losses.ce, encoders.Linear, emsize=1024, nhid=2048, nlayers=6, nhead=4,
                       dropout=0.0, epochs=1, steps_per_epoch=steps + 3, batch_size=1000, bptt=T, lr=1e-4, warmup_epochs=1,
                       y_encoder_generator=encoders.get_Canonical(C), extra_prior_kwargs_dict=dict(KW, fuse_x_y=False),
                       single_eval_pos_gen=T - 1, gpu_device='cuda:0')
    (x, y), tgt = next(iter(tr.dl))
    for _ in range(3):
        tr.step((x, y), tgt, T - 1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        tr.step((x, y), tgt, T - 1)
    torch.cuda.synchronize()
    pre = (time.perf_counter() - t0) / steps
    it = iter(tr.dl)
    for _ in range(3):
        (x, y), tgt = next(it)
        tr.step((x, y), tgt, T - 1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        (x, y), tgt = next(it)
        tr.step((x, y), tgt, T - 1)
    torch.cuda.synchronize()
    fed = (time.perf_counter() - t0) / steps
    print(f"Trainer.step emsize 1024 nhead 4 6 layers B=1000 T=26: pre-drawn batch {pre * 1e3:.2f} ms/step, "
          f"sampled by the prefetching loader {fed * 1e3:.2f} ms/step")


def short_train(steps):
    import transformerscandobayesianinference_b200 as pfn
    mods = pfn.install_dropin()
    import priors.stroke  # noqa: F401  (the drop-in module, as the notebook imports it)
    encoders, train_mod = mods["encoders"], mods["train"]
    torch.manual_seed(0)
    t0 = time.perf_counter()
    res = train_mod.train(sys.modules["priors.stroke"].DataLoader, train_mod.Losses.ce, encoders.Linear, emsize=1024, nhead=4,
                          warmup_epochs=5, nhid=2048, y_encoder_generator=encoders.get_Canonical(5), lr=.0001, epochs=1,
                          single_eval_pos_gen=T - 1, extra_prior_kwargs_dict=dict(KW, fuse_x_y=False), bptt=T, nlayers=6,
                          dropout=0.0, steps_per_epoch=steps, batch_size=1000)
    torch.cuda.synchronize()
    print(f"train(priors.stroke.DataLoader, ...) notebook settings, 1 epoch x {steps} steps: {time.perf_counter() - t0:.1f} s, "
          f"final loss {res[0]:.4f}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--train-steps", type=int, default=10)
    ap.add_argument("--reference-dir", default=None, help="reference checkout: also time its priors/stroke.py on the host")
    a = ap.parse_args()
    if a.reference_dir:
        time_reference(1000, a.reference_dir)
    if not torch.cuda.is_available():
        print("no CUDA device: device timings skipped")
        return
    from transformerscandobayesianinference_b200.priors import stroke
    print(f"device: {torch.cuda.get_device_name(0)}")
    for B in (1000, 512):
        med, best = time_device(stroke, B, a.iters)
        mb = T * B * F * 4 / 1e6
        print(f"device get_batch B={B} T={T} F={F}: median {med:.3f} ms, best {best:.3f} ms ({mb:.0f} MB of x, "
              f"{mb / 1e3 / (med / 1e3):.0f} GB/s effective)")
        print(f"  kernels (torch.profiler, per call, B={B}):")
        profile_kernels(stroke, B)
    time_steps(stroke, a.steps)
    if a.train_steps > 0:
        short_train(a.train_steps)


if __name__ == "__main__":
    main()
