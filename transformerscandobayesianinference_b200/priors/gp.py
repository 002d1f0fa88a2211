"""`priors.gp` (reference priors/gp.py): functions drawn from a Gaussian process with a unit-amplitude RBF kernel of fixed
length scale and no noise, and its exact-GP baseline `evaluate`.  The reference calls sklearn's GaussianProcessRegressor
once per dataset (sampling) and once per dataset and prefix (evaluation); here both are one launch of the fp64 kernels
of csrc/regression_baselines.cu, and nothing imports sklearn (`get_gp`, which returns a sklearn estimator, is not
provided).

Sampling matches the reference in distribution, not in its random stream: x ~ U[0,1) and the normals are drawn with
torch on the device, and y = P L z comes from a pivoted Cholesky of K that stops at the numerical rank, as exact as
numpy's SVD-based multivariate_normal that sklearn uses, and like it without any jitter.  T <= 128 (the T x T fp64
matrix of a dataset lives in one SM's shared memory)."""
import math
import time

import torch

from .. import _lib as L
from ..utils import default_device
from .utils import get_batch_to_dataloader, on_requested_device

length_scale_sampling_gp = .6
_ALPHA = 1e-10                  # sklearn GaussianProcessRegressor's default alpha, added to the training diagonal
_VAR_EPS = 1e-6                 # torch GaussianNLLLoss's default eps: the variance is clamped at it
_KERNEL = "priors.gp runs on the sm_90a exact-GP kernels"


def _check_len(T, who):
    if T > L.GP_FIT_MAX_T:
        raise ValueError(f"priors.gp.{who}: sequence length {T} exceeds {L.GP_FIT_MAX_T} (one dataset's T x T fp64 "
                         "kernel matrix lives in shared memory)")


@torch.no_grad()
def get_batch(batch_size, seq_len, num_features, noisy_std=None, device=default_device, x=None, z=None):
    """-> x [T,B,F], y [T,B], y (reference :19-34).  As in the reference, `noisy_std` is the kernel's LENGTH SCALE
    (`get_gp(noisy_std)`, :28; None or 0 -> .6).  Optional `x` [B,T,F] ~ U[0,1) and `z` [B,T] ~ N(0,1) replace the
    device draws (z[b, k] scales the k-th pivot column of the factor)."""
    _check_len(seq_len, "get_batch")
    length_scale = noisy_std or length_scale_sampling_gp
    dev = L.compute_device(device, _KERNEL)
    if x is not None:
        assert x.shape == (batch_size, seq_len, num_features)
        x = x.to(dev, torch.float32).contiguous()
    else:
        x = torch.rand(batch_size, seq_len, num_features, device=dev)
    if z is not None:
        assert z.shape == (batch_size, seq_len)
        z = z.to(dev, torch.float32).contiguous()
    else:
        z = torch.randn(batch_size, seq_len, device=dev)
    y = torch.empty(batch_size, seq_len, device=dev)
    rank = torch.empty(batch_size, dtype=torch.int32, device=dev)
    L.exact_gp_sample(x, z, length_scale, y, rank)
    x_t, y_t = on_requested_device(device, x.transpose(0, 1), y.transpose(0, 1))
    return x_t, y_t, y_t


DataLoader = get_batch_to_dataloader(get_batch)
DataLoader.num_outputs = 1


def _first_rejected_t(xb, yb):
    """Per dataset, the first prefix t whose sklearn fit or predict would reject a non-finite input (T: none): rows < t and
    row t of x are validated at t, rows < t of y."""
    T = xb.shape[1]
    idx = torch.arange(T, device=xb.device)
    rx = torch.where(torch.isfinite(xb).all(-1), T, idx).amin(1)
    ry = torch.where(torch.isfinite(yb), T, idx).amin(1)
    t_x = torch.where(rx < T, rx.clamp_min(1), T)
    t_y = torch.where(ry + 1 < T, ry + 1, T)
    return torch.minimum(t_x, t_y)


@torch.no_grad()
def evaluate(x, y, y_non_noisy, use_mse=False, length_scale=length_scale_sampling_gp):
    """Exact-GP baseline (reference :41-62): for each t = 1 .. T-1 and dataset b, the GP with kernel RBF(length_scale)
    and alpha = 1e-10 conditioned on rows < t predicts row t, scored against y (not y_non_noisy, as in the reference) by
    torch's GaussianNLLLoss(full=True) with the latent variance clamped at 1e-6, or by the squared error of the mean.
    x [T,B,F], y [T,B] on any device; runs on the CUDA device that holds x (the current one for CPU tensors).  Returns
    (tensor([0., mean_b loss[1, b], ...]) fp64 on the CPU, seconds).  Raises ValueError, naming the dataset and t, where
    the reference's sklearn raises: a non-finite input, or a kernel matrix whose Cholesky factor fails."""
    start = time.time()
    _check_len(len(x), "evaluate")
    length_scale = length_scale or length_scale_sampling_gp
    dev = L.compute_device(x.device, _KERNEL)
    xb = x.to(dev, torch.float32).transpose(0, 1).contiguous()        # [B,T,F]
    yb = y.to(dev, torch.float32).transpose(0, 1).contiguous()        # [B,T]
    B, T, _ = xb.shape
    mean = torch.empty(B, T, dtype=torch.float64, device=dev)
    var = torch.empty_like(mean)
    status = torch.empty(B, dtype=torch.int32, device=dev)
    L.exact_gp_evaluate(xb, yb, length_scale, _ALPHA, mean, var, status)
    rejected = _first_rejected_t(xb, yb)
    failed = torch.minimum(rejected, torch.where(status > 0, status.long(), T))
    t_fail = int(failed.min())
    if t_fail < T:
        b = int((failed == t_fail).nonzero()[0])
        if int(rejected[b]) == t_fail:          # sklearn validates its inputs before it factors anything
            raise ValueError(f"priors.gp.evaluate: dataset {b}, t={t_fail}: a non-finite input (sklearn rejects it in "
                             f"the fit on rows < {t_fail} or in the predict of row {t_fail})")
        raise ValueError(f"priors.gp.evaluate: dataset {b}, t={t_fail}: the kernel matrix of the fit on rows < {t_fail} "
                         "is not positive definite")
    target = yb[:, 1:].double()
    if use_mse:
        per_t = (mean[:, 1:] - target) ** 2
    else:
        v = var[:, 1:].clamp_min(_VAR_EPS)
        per_t = 0.5 * (torch.log(v) + (mean[:, 1:] - target) ** 2 / v) + 0.5 * math.log(2 * math.pi)
    losses = torch.cat([torch.zeros(1, dtype=torch.float64, device=dev), per_t.mean(0)])
    return losses.cpu(), time.time() - start
