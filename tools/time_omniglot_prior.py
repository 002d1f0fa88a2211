"""Time priors.omniglot: one device batch at the FewShotOmniglot notebook's shapes (5-way 5-shot, 28 x 28, B = 1000 and
B = 100, default and Jonas episodes, translations on) over the synthetic bank of tests/test_gpu_omniglot_prior.py, with
CUDA events for the call and torch.profiler for the kernel, and the achieved write rate (x, y and target_y).  Given a
reference checkout, also the reference loader's host time per batch over the same bank written as a PNG tree (this needs
no GPU; PIL and torchvision must import).

    python tools/time_omniglot_prior.py [--iters 50] [--reference-dir <reference checkout>]
"""
import argparse
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gpu_timing import card, event_times, kernel_seconds  # noqa: E402

S, N_WAY, K_SHOT = 28, 5, 5
T = N_WAY * K_SHOT + 1


def written_bytes(B):
    return T * B * (S * S * 4 + 8 + 8)


def time_device(omniglot, bank, B, jonas, iters):
    desc = omniglot.episode_desc(bank, B, N_WAY, K_SHOT, train=True, jonas_style=jonas, translations=True)
    def calls():
        for _ in range(iters):
            omniglot.sample_episodes(bank, desc)
    ms = [1e3 * s for s in event_times(lambda: omniglot.sample_episodes(bank, desc), iters, warmup=5)]
    kernels = kernel_seconds(calls)
    kern = [(s, n) for name, (s, n) in kernels.items() if "omniglot_episode_kernel" in name]
    us = kern[0][0] / kern[0][1] * 1e6 if kern else float("nan")
    return statistics.median(ms), min(ms), us


def time_reference(tm, reference_dir, batches):
    from make_omniglot_golden import load_reference_omniglot, sorted_walk
    images, alphabets = tm.synthetic_bank()
    ref = load_reference_omniglot(os.path.abspath(reference_dir))
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        tm.write_tree(tmp, images, alphabets)
        os.chdir(tmp)
        try:
            for jonas in (False, True):
                np.random.seed(0)
                t0 = time.perf_counter()
                with sorted_walk():
                    dl = ref.DataLoader(num_steps=batches, batch_size=1000, seq_len=T, num_features=S * S, num_outputs=N_WAY,
                                        train=True, translations=True, jonas_style=jonas)
                t1 = time.perf_counter()
                per = []
                it = iter(dl)
                for _ in range(batches):
                    t2 = time.perf_counter()
                    next(it)
                    per.append(time.perf_counter() - t2)
                print(f"reference loader, {'Jonas' if jonas else 'default'} mode, B=1000: construction {t1 - t0:.1f} s, "
                      f"per batch {statistics.median(per):.2f} s (median of {batches}; one Python thread, "
                      f"{os.cpu_count()} cores visible, torch threads {torch.get_num_threads()})", flush=True)
        finally:
            os.chdir(cwd)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reference-dir", default=None)
    ap.add_argument("--reference-batches", type=int, default=3)
    a = ap.parse_args()
    from make_omniglot_golden import _test_module
    tm = _test_module()
    if a.reference_dir:
        time_reference(tm, a.reference_dir, a.reference_batches)
    print(f"device: {card('time_omniglot_prior')}")
    from transformerscandobayesianinference_b200.priors import omniglot
    bank = omniglot.Bank(*tm.synthetic_bank())
    for B in (1000, 100):
        for jonas in (False, True):
            med, best, us = time_device(omniglot, bank, B, jonas, a.iters)
            mb = written_bytes(B) / 1e6
            print(f"B={B} {'Jonas  ' if jonas else 'default'}: call median {med * 1e3:.1f} us, best {best * 1e3:.1f} us (CUDA events, "
                  f"{a.iters} calls); omniglot_episode_kernel {us:.1f} us (torch.profiler); {mb:.1f} MB written, "
                  f"{mb / 1e3 / (us * 1e-6):.0f} GB/s over the kernel time", flush=True)


if __name__ == "__main__":
    main()
