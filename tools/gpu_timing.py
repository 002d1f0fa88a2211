"""How the measurement scripts under tools/ time GPU work and name the card they ran on.

Every number in DESIGN.md §3.1 is taken through these four functions, so one policy holds for all of them: the card is
read in the same run, each timed sample is bracketed by CUDA events on the current stream after a synchronise, and
kernel times come from torch.profiler in a pass of their own."""
import subprocess

import torch


def card(tool):
    """One line naming the card: name, power limit and max SM clock.  Raises SystemExit naming `tool` when there is no
    CUDA device (nothing is timed on the host alone); says so in the line when nvidia-smi cannot be read."""
    if not torch.cuda.is_available():
        raise SystemExit(f"{tool} needs a CUDA device (nothing is timed on the host alone)")
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        return f"{torch.cuda.get_device_name()}, power limit not read, max SM clock not read"


def event_times(fn, reps, warmup=1, calls=1):
    """Sorted seconds per call of fn(): `warmup` calls, a synchronise, then `reps` samples, each one CUDA-event bracket
    on the current stream around `calls` calls (divided by `calls`) followed by a synchronise."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(calls):
            fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3 / calls)
    return sorted(times)


def kernel_seconds(fn):
    """{kernel name: (total device seconds, launches)} of every CUDA kernel that one call of fn() runs, from
    torch.profiler with CUDA activities (synchronised before and after the call)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            s, n = kernels.get(ev.name, (0.0, 0))
            kernels[ev.name] = (s + ev.device_time_total / 1e6, n + 1)
    return kernels


def attention_pairs(T, sep):
    """(query, key) pairs the masked attention computes: every row attends the sep train keys, rows >= sep also their
    own key."""
    return T * sep + (T - sep)
