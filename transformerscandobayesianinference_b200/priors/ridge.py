"""`priors.ridge` (reference priors/ridge.py): noisy linear functions with N(0, .1^2) weights (:12-18), and the Ridge
baseline `evaluate` (:23-34), whose per-prefix sklearn fits run as one launch of csrc/regression_baselines.cu."""
import time

import torch

from .. import _lib as L
from .utils import get_batch_to_dataloader

_KERNEL = "priors.ridge.evaluate fits with the sm_90a ridge kernel"


def get_batch(batch_size, seq_len, num_features, noisy_std=.1, device='cpu'):
    m = torch.normal(0., .1, size=(batch_size, num_features), device=device)
    x = torch.rand(seq_len, batch_size, num_features, device=device)
    y_non_noisy = torch.einsum('bf,tbf->tb', m, x)
    y = y_non_noisy + torch.normal(torch.zeros_like(y_non_noisy), noisy_std)
    return x, y, y_non_noisy


DataLoader = get_batch_to_dataloader(get_batch)
DataLoader.num_outputs = 1


@torch.no_grad()
def evaluate(x, y, y_non_noisy, alpha=0.):
    """For each t = 1 .. T-1 and dataset b: sklearn's Ridge(alpha) (with intercept) fitted to rows < t of (x[:, b], y[:, b])
    predicts row t, scored by its squared error against y_non_noisy[t, b].  x [T,B,F], y and y_non_noisy [T,B] on any
    device; the fits run on the CUDA device that holds x (the current one for CPU tensors).  Returns
    (tensor([0., mean_b err[1, b], ..., mean_b err[T-1, b]]) fp64 on the CPU, seconds), like the reference.

    With alpha = 0 a prefix whose centred rows are rank deficient (always when t <= F) gets the minimum-norm solution,
    singular values at or below max(t, F) eps s_max counting as zero (numpy lstsq's cutoff); sklearn reaches the same
    solution through its SVD fallback when its Cholesky fails."""
    start = time.time()
    alpha = float(alpha)
    if not alpha >= 0.0:
        raise ValueError(f"priors.ridge.evaluate: alpha={alpha} must be >= 0")
    F = x.shape[2]
    if F > L.RIDGE_MAX_F:
        raise ValueError(f"priors.ridge.evaluate: {F} features exceed the kernel's limit of {L.RIDGE_MAX_F}")
    dev = L.compute_device(x.device, _KERNEL)
    xb, yb, tb = (v.to(dev, torch.float32).transpose(0, 1).contiguous() for v in (x, y, y_non_noisy))
    B, T, _ = xb.shape
    pred = torch.empty(B, T, dtype=torch.float64, device=dev)
    sq_err = torch.empty_like(pred)
    L.ridge_prefix(xb, yb, tb, alpha, pred, sq_err)
    losses = torch.cat([torch.zeros(1, dtype=torch.float64, device=dev), sq_err[:, 1:].mean(0)])
    return losses.cpu(), time.time() - start
