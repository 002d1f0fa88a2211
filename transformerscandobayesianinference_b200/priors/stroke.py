"""`priors.stroke` (reference priors/stroke.py): synthetic handwriting for few-shot image classification.

Each dataset has `num_outputs` classes; a class is 1..3 straight strokes (start, length, direction) drawn by rejection so
that every stroke ends inside the canvas.  Each image of the sequence is its class's strokes drawn with a random width,
offset and end-point jitter, the ink filled with U{200..254}, blurred with PIL's GaussianBlur(0.2) and scaled to [0, 1].

Where the reference draws every image in Python with PIL (26 000 per batch of the Omniglot notebook), the images here are
rasterised and blurred by csrc/stroke_prior.cu, one warp per image, bit-exactly like Pillow's `ImageDraw.line` and
`GaussianBlur` for the same end points, width and fill; x is written straight into the [seq_len, batch, size^2] layout.
The random numbers are counter-based hashes of one seed per batch drawn from torch's CPU generator, so a batch is
reproducible under `torch.manual_seed` and costs no device sync; the class table is drawn with device torch ops.  The
distribution is the reference's, the individual draws are not (Python's `random` and numpy streams are not replayed).

`mnist_prior`, which returns callables producing PIL images, is not provided: it is not on the training path.
"""
import math
import os
import random

import torch

from .. import _lib as L
from ..utils import default_device
from .utils import check_flag, get_batch_to_dataloader, on_requested_device

# mnist_prior's keyword defaults (reference :9-10), as fractions of the image side
PRIOR_DEFAULTS = dict(min_max_strokes=(1, 3), min_max_len=(5 / 28, 20 / 28), min_max_start=(2 / 28, 25 / 28),
                      min_max_width=(1 / 28, 4 / 28), max_offset=4 / 28, max_target_offset=2 / 28)
MAX_ITERS = 256          # rejection draws per stroke before the batch is refused (the reference loops without a bound)


class StrokeRejectionError(RuntimeError):
    pass


def normalize(x):
    """Per-image standardisation with torch's unbiased std (reference :74-75)."""
    return (x - x.mean()) / (x.std() + .000001)


def stroke_desc(size, num_outputs, max_iters=MAX_ITERS, **kwargs):
    """The integer ranges of the reference's `random.randint` calls for an image side `size` (reference :13-16, :26-28,
    :49-54), validated on the host.  Unknown keywords raise TypeError like `mnist_prior(**kwargs)` does."""
    unknown = set(kwargs) - set(PRIOR_DEFAULTS)
    if unknown:
        raise TypeError(f"priors.stroke: unexpected keyword argument(s) {sorted(unknown)}")
    kw = dict(PRIOR_DEFAULTS, **kwargs)
    d = L.StrokeDesc()
    d.S, d.C, d.max_iters = size, num_outputs, max_iters
    d.strokes_min, d.strokes_max = int(kw["min_max_strokes"][0]), int(kw["min_max_strokes"][1])
    d.len_min, d.len_max = int(size * kw["min_max_len"][0]), int(size * kw["min_max_len"][1])
    d.start_min, d.start_max = int(size * kw["min_max_start"][0]), int(size * kw["min_max_start"][1])
    d.width_min, d.width_max = int(size * kw["min_max_width"][0]), int(size * kw["min_max_width"][1])
    d.offset_min, d.offset_max = int(-size * kw["max_offset"]), int(size * kw["max_offset"])
    d.jitter_min, d.jitter_max = int(-size * kw["max_target_offset"]), int(size * kw["max_target_offset"])
    for name, lo, hi in (("min_max_strokes", d.strokes_min, d.strokes_max), ("min_max_len", d.len_min, d.len_max),
                         ("min_max_start", d.start_min, d.start_max), ("min_max_width", d.width_min, d.width_max),
                         ("max_offset", d.offset_min, d.offset_max), ("max_target_offset", d.jitter_min, d.jitter_max)):
        if lo > hi:
            raise ValueError(f"priors.stroke: {name}={kw[name]!r} gives the empty integer range [{lo}, {hi}] at size {size}")
    if d.strokes_min < 1 or d.strokes_max > L.STROKE_MAX_STROKES:
        raise ValueError(f"priors.stroke: min_max_strokes={kw['min_max_strokes']!r} must lie in [1, {L.STROKE_MAX_STROKES}]")
    if not 1 <= size <= L.STROKE_MAX_SIDE:
        raise ValueError(f"priors.stroke: image side {size} outside [1, {L.STROKE_MAX_SIDE}] "
                         f"(num_features = side^2 <= {L.STROKE_MAX_SIDE ** 2})")
    if num_outputs < 1:
        raise ValueError(f"priors.stroke: num_outputs={num_outputs} must be >= 1")
    return d


def _reject(d, kw):
    kw = dict(PRIOR_DEFAULTS, **kw)
    raise StrokeRejectionError(
        f"priors.stroke: a class stroke found no end point inside [0, {d.S - 1}]^2 in {d.max_iters} rejection draws; "
        f"min_max_len={kw['min_max_len']!r} (lengths {d.len_min}..{d.len_max}) is too long for "
        f"min_max_start={kw['min_max_start']!r} (starts {d.start_min}..{d.start_max}) at size {d.S}")


def class_table(batch_size, seq_len, num_outputs, only_train_for_last_idx, device):
    """Class of every position, int64 [seq_len, batch_size], with device ops (reference :97-105).  Last-index mode: each class
    exactly (seq_len - 1) / num_outputs times among the first seq_len - 1 positions in shuffled order, then a uniform
    class; otherwise uniform classes everywhere."""
    if not only_train_for_last_idx:
        return torch.randint(0, num_outputs, (seq_len, batch_size), device=device)
    reps = (seq_len - 1) // num_outputs
    last = torch.randint(0, num_outputs, (1, batch_size), device=device)
    if reps == 0:
        return last
    order = torch.rand(batch_size, seq_len - 1, device=device).argsort(1)      # a uniform permutation per dataset
    return torch.cat([(order // reps).t(), last], 0)


def sample_geometry(batch_size, desc, seed, device):
    """(geom [B, C, strokes_max, 4] int32 (start x, start y, length, active), turns [B, C, strokes_max] fp64, cap flag)"""
    geom = torch.empty(batch_size, desc.C, desc.strokes_max, 4, dtype=torch.int32, device=device)
    turns = torch.empty(batch_size, desc.C, desc.strokes_max, dtype=torch.float64, device=device)
    flag = torch.zeros(1, dtype=torch.int32, device=device)
    L.stroke_geometry(desc, seed, geom, turns, flag)
    return geom, turns, flag


@torch.no_grad()
def get_batch(batch_size, seq_len, num_features=None, noisy_std=None, only_train_for_last_idx=False, normalize_x=False,
              num_outputs=2, use_saved_from=None, device=default_device, **kwargs):
    """-> x [seq_len, B, num_features] fp32, y [seq_len, B] int64 (the classes), target_y [seq_len, B] int64 (reference
    :80-114).  With `only_train_for_last_idx` every target but the last position's is -100.  `noisy_std` is accepted and
    ignored, as in the reference.  Keywords of the reference's `mnist_prior` (min_max_len, ...) pass through."""
    if use_saved_from is not None:
        directory = os.path.join(use_saved_from, f'len_{seq_len}_out_{num_outputs}_features_{num_features}_bs_{batch_size}')
        filename = random.choice(os.listdir(directory))
        return torch.load(os.path.join(directory, filename))

    size = math.isqrt(num_features)
    assert size * size == num_features, 'num_features needs to be the square of an integer.'
    if only_train_for_last_idx:
        assert (seq_len - 1) % num_outputs == 0
    desc = stroke_desc(size, num_outputs, **kwargs)
    dev = L.compute_device(device, "priors.stroke draws its images with the sm_90a stroke kernels")
    seed = L.draw_seed()

    with L.on_device(dev):
        y = class_table(batch_size, seq_len, num_outputs, only_train_for_last_idx, dev)
        geom, turns, flag = sample_geometry(batch_size, desc, seed, dev)
        x = torch.empty(seq_len, batch_size, num_features, dtype=torch.float32, device=dev)
        L.stroke_render(desc, seed, y.to(torch.int32).contiguous(), geom, turns, x, normalize_x)
        if only_train_for_last_idx:
            target_y = torch.full_like(y, -100)
            target_y[-1] = y[-1]
        else:
            target_y = y
        check_flag(flag, lambda: _reject(desc, kwargs))
    return on_requested_device(device, x, y, target_y)


DataLoader = get_batch_to_dataloader(get_batch)
DataLoader.num_outputs = 2
