"""Prior -> DataLoader adapter and small sampling helpers (reference priors/utils.py).  No plotting imports: the
reference pulls in matplotlib at module import (priors/utils.py:10-11), which is not part of the hot path."""
import random

import numpy as np
import scipy.stats as stats
import torch
from torch import nn

from .. import _lib as L
from ..utils import set_locals_in_self
from .prior import PriorDataLoader


class _Deferred:
    """Registry of device-side validity checks that a sampler could not finish without a host sync (e.g. the Cholesky
    pivot flags of priors.fast_gp).  While `active`, `check_flag` appends a zero-argument callable instead of syncing; the
    prefetching loader runs them when the batch is handed to the consumer — a full step later, when the flags have long
    been copied to pinned host memory, so nothing stalls."""
    active = False
    pending = []

    @classmethod
    def collect(cls):
        out, cls.pending = cls.pending, []
        return out


def check_flag(flag, on_set, may_defer=True):
    """Calls `on_set()` when the int32 device tensor `flag` [1] is non-zero.  While a loader defers (and `may_defer`), the
    flag travels to pinned host memory behind the work on the current stream and is looked at when the batch is handed
    over; otherwise it is read at once (a host sync).  Returns whether the check was deferred."""
    if not (may_defer and _Deferred.active):
        if int(flag.item()) != 0:
            on_set()
        return False
    flag_host = torch.empty(1, dtype=torch.int32, pin_memory=True)
    flag_host.copy_(flag, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream(flag.device))

    def resolve():
        ev.synchronize()
        if int(flag_host[0]) != 0:
            on_set()
    _Deferred.pending.append(resolve)
    return True


def again_after_deferred_checks(fn):
    """Calls `fn()` at once and, while a loader defers and checks are pending, once more at hand-off after them (a check
    may rewrite a sampler's output in place, e.g. fast_gp's jitter escalation).  So what `fn` writes is valid at once and
    final after hand-off; anything derived from it before hand-off (inside the loader's `_produce`) may be stale."""
    fn()
    if _Deferred.active and _Deferred.pending:
        _Deferred.pending.append(fn)


def on_requested_device(device, *tensors):
    """A sampler's outputs, copied to `device` when the caller asked for a non-CUDA one (the sampler ran on CUDA)."""
    dev = torch.device(device)
    return tensors if dev.type == 'cuda' else tuple(t.to(dev) for t in tensors)


def prefetch_enabled():
    import os
    return os.environ.get("PFN_B200_PREFETCH", "1") != "0" and torch.cuda.is_available()


def _tensors_of(obj):
    if torch.is_tensor(obj):
        yield obj
    elif isinstance(obj, (tuple, list)):
        for o in obj:
            yield from _tensors_of(o)


def get_batch_to_dataloader(get_batch_method_):
    """Wrap a `get_batch(batch_size, seq_len, num_features, ...) -> (x, y, target_y)` function into a loader class
    that yields `num_steps` freshly sampled batches per epoch as `((x, y), target_y)` (reference :14-42)."""

    class DL(PriorDataLoader):
        get_batch_method = get_batch_method_

        # `num_features` may be a class attribute set before instantiation when it is not part of the kwargs.
        def __init__(self, num_steps, fuse_x_y=False, **get_batch_kwargs):
            set_locals_in_self(locals())
            self.num_features = get_batch_kwargs.get('num_features') or self.num_features
            self.num_outputs = get_batch_kwargs.get('num_outputs') or self.num_outputs
            print('DataLoader.__dict__', self.__dict__)

        @staticmethod
        def gbm(*args, fuse_x_y=True, **kwargs):
            x, y, target_y = get_batch_method_(*args, **kwargs)
            if fuse_x_y:
                shifted = torch.cat([torch.zeros_like(y[:1]), y[:-1]], 0).unsqueeze(-1).float()
                return torch.cat([x, shifted], -1), target_y
            return (x, y), target_y

        def __len__(self):
            return self.num_steps

        def _produce(self):
            return self.gbm(**self.get_batch_kwargs, fuse_x_y=self.fuse_x_y)

        def __iter__(self):
            """Yields `num_steps` fresh batches.  On CUDA the NEXT batch is sampled on a low-priority side stream while
            the consumer works on the current one (sampling does not depend on the weights), and deferred sampler
            checks are resolved at hand-off.  The reference builds every batch synchronously (priors/utils.py:36-37)."""
            if not prefetch_enabled():
                return iter(self._produce() for _ in range(self.num_steps))
            return self._iter_prefetch()

        def _iter_prefetch(self):
            side = getattr(self, '_side_stream', None)
            if side is None:
                dev = L.compute_device(self.get_batch_kwargs.get('device'), "the prefetching loader samples on a side stream")
                side = self._side_stream = torch.cuda.Stream(device=dev, priority=0)
                self._side_device = dev

            def launch():
                prev = _Deferred.active
                _Deferred.active = True
                try:
                    side.wait_stream(torch.cuda.current_stream(self._side_device))   # allocator reuse / ordering w.r.t. the consumer
                    with torch.cuda.stream(side):
                        batch = self._produce()
                        ev = torch.cuda.Event()
                        ev.record(side)
                    checks = _Deferred.collect()
                finally:
                    _Deferred.active = prev
                return batch, ev, checks

            nxt = launch() if self.num_steps > 0 else None
            for i in range(self.num_steps):
                batch, ev, checks = nxt
                nxt = launch() if i + 1 < self.num_steps else None
                cur = torch.cuda.current_stream(self._side_device)
                cur.wait_event(ev)
                for t in _tensors_of(batch):
                    if t.is_cuda:
                        t.record_stream(cur)
                for chk in checks:
                    chk()
                yield batch

    return DL


trunc_norm_sampler_f = lambda mu, sigma: lambda: stats.truncnorm((0 - mu) / sigma, (1 - mu) / sigma, loc=mu, scale=sigma).rvs(1)[0]
beta_sampler_f = lambda a, b: lambda: np.random.beta(a, b)
gamma_sampler_f = lambda a, b: lambda: np.random.gamma(a, b)
uniform_sampler_f = lambda a, b: lambda: np.random.uniform(a, b)
uniform_int_sampler_f = lambda a, b: lambda: np.random.randint(a, b)
zipf_sampler_f = lambda a, b, c: lambda: min(b + np.random.zipf(a), c)
scaled_beta_sampler_f = lambda a, b, scale, minimum: lambda: minimum + round(beta_sampler_f(a, b)() * (scale - minimum + 1) - 0.5)


def normalize_data(data):
    """Zero mean / unit (unbiased) std over dim 0, eps 1e-6 (reference :73-78)."""
    return (data - data.mean(0)) / (data.std(0) + .000001)


def normalize_by_used_features_f(x, num_features_used, num_features):
    return x / (num_features_used / num_features)


class Binarize(nn.Module):
    """1 where x exceeds the (lower) median of the WHOLE tensor (reference :85-91)."""

    def __init__(self, p=0.5):
        super().__init__()
        self.p = p

    def forward(self, x):
        return (x > torch.median(x)).float()


def order_by_y(x, y):
    """Sort the sequence by (+/-) y of the first dataset, then interleave the two halves (reference :94-100)."""
    order = torch.argsort(y if random.randint(0, 1) else -y, dim=0)[:, 0, 0]
    order = order.reshape(2, -1).transpose(0, 1).reshape(-1)
    return x[order], y[order]
