"""`priors.fast_gp` (reference priors/fast_gp.py): one GP-prior draw per dataset,
    x ~ U[0,1)^(B x T x F),  y = chol(outputscale * RBF(x, x; lengthscale) + noise * I) z,  z ~ N(0, I),
sampled by the fused CUDA kernel csrc/gp_sampler.cu (kernel build + blocked fp32 Cholesky + L z in one pass)
instead of gpytorch's lazy kernel -> cuSOLVER potrf -> bmm chain (reference :13-32,48-56).

gpytorch semantics kept: default hyperparameters (:40), tuple/list hyperparameters (:37-38), the RNG order
`rand` (x) then `randn` (z), and psd_safe_cholesky's jitter escalation (1e-6, 1e-5, 1e-4 added to the whole
batch's diagonal, then NotPSD error).  `fast_computations` is accepted and ignored: the kernel always computes
the exact Cholesky root (what the notebook's `(False, False, False)` setting selects).
"""
import math

import torch

from .. import _lib as L
from ..utils import default_device
from .utils import check_flag, get_batch_to_dataloader, on_requested_device

_JITTERS = (0.0, 1e-6, 1e-5, 1e-4)
_KERNEL = "priors.fast_gp samples with the sm_90a GP kernel"


class NotPSDError(RuntimeError):
    pass


def sample_gp(x, z, lengthscale, outputscale, noise, kernel_type=L.KERNEL_RBF, return_factor=False, may_defer=True):
    """x [B,T,F], z [B,T] on a CUDA device; lengthscale [B,F], outputscale [B], noise [B] -> y [B,T].

    The pivot flags of the jitter-0 factorisation go through `check_flag`: while a loader defers (and `may_defer`), they
    are looked at when the batch is handed to the consumer, a step later, with no host sync here.  Only if a pivot failed
    is the whole batch re-factored with gpytorch's jitter escalation, overwriting y in place (every view handed out stays
    valid).  With `return_factor` the check is immediate and the factor of the jitter that succeeded is returned too."""
    Bn, T, F = x.shape
    dev = x.device
    ldw = (T + 3) // 4 * 4
    y = torch.empty(Bn, T, device=dev, dtype=torch.float32)
    work = torch.empty(Bn, T, ldw, device=dev, dtype=torch.float32)
    info = torch.empty(Bn, device=dev, dtype=torch.int32)
    L.gp_sample(x, z, lengthscale, outputscale, noise, _JITTERS[0], kernel_type, y, work, info)

    def escalate():
        nonlocal work
        if work is None:
            work = torch.empty(Bn, T, ldw, device=dev, dtype=torch.float32)
        for jitter in _JITTERS[1:]:
            L.gp_sample(x, z, lengthscale, outputscale, noise, jitter, kernel_type, y, work, info)
            if not bool(info.any().item()):
                return
        raise NotPSDError(f"kernel matrix not positive definite even with jitter {_JITTERS[-1]:g} "
                          f"(first failing pivots: {info[info > 0][:8].tolist()})")

    if check_flag(info.max().reshape(1), escalate, may_defer and not return_factor):
        work = None             # B T^2 floats not held through the step before the check; escalate allocates them again
    return (y, torch.tril(work[:, :, :T].transpose(1, 2))) if return_factor else y


def _hps_to_dict(hyperparameters):
    if isinstance(hyperparameters, (tuple, list)):
        return {"noise": hyperparameters[0], "outputscale": hyperparameters[1], "lengthscale": hyperparameters[2]}
    if hyperparameters is None:
        return {"noise": .1, "outputscale": .1, "lengthscale": .1}
    return hyperparameters


@torch.no_grad()
def get_batch(batch_size, seq_len, num_features, device=default_device, hyperparameters=None, equidistant_x=False,
              x=None, z=None):
    """-> x [T,B,F], y [T,B], target_y [T,B] (= y) on `device` (reference :36-58).

    Extension (defaults keep the reference signature): `x` [B,T,F] ~ U[0,1) and `z` [B,T] ~ N(0,1) may be supplied by
    the caller — e.g. drawn on the host and kept in pinned memory — instead of being drawn on the device; they are
    copied to the device asynchronously."""
    hps = _hps_to_dict(hyperparameters)
    dev = L.compute_device(device, _KERNEL)
    if x is not None:
        assert x.shape == (batch_size, seq_len, num_features)
        x = x.to(dev, torch.float32, non_blocking=True).contiguous()
    elif equidistant_x:
        assert num_features == 1
        x = torch.linspace(0, 1., seq_len, device=dev).view(1, seq_len, 1).repeat(batch_size, 1, 1)
    else:
        x = torch.rand(batch_size, seq_len, num_features, device=dev)
    if z is not None:
        assert z.shape == (batch_size, seq_len)
        z = z.to(dev, torch.float32, non_blocking=True).contiguous()
    else:
        z = torch.randn(batch_size, seq_len, device=dev)
    ls = torch.full((batch_size, num_features), float(hps["lengthscale"]), device=dev)
    os_ = torch.full((batch_size,), float(hps["outputscale"]), device=dev)
    noise = torch.full((batch_size,), float(hps["noise"]), device=dev)
    y = sample_gp(x, z, ls, os_, noise, L.KERNEL_RBF)
    x_t, y_t = on_requested_device(device, x.transpose(0, 1), y.transpose(0, 1))
    return x_t, y_t, y_t


DataLoader = get_batch_to_dataloader(get_batch)
DataLoader.num_outputs = 1


class _Predictive:
    """The slice of gpytorch's MultivariateNormal the reference touches (priors/fast_gp.py:102-115): `.mean`,
    `.covariance_matrix`, `.variance`, `.log_prob(y)` for batched predictions at ONE test point per dataset."""

    def __init__(self, mean, var):
        self.mean = mean                       # [B, 1]
        self.variance = var                    # [B, 1]
        self.covariance_matrix = var.unsqueeze(-1)   # [B, 1, 1]

    def log_prob(self, value):
        v = value.reshape(self.mean.shape).to(self.mean.dtype)
        return (-0.5 * (math.log(2 * math.pi) + torch.log(self.variance) + (v - self.mean) ** 2 / self.variance)).sum(-1)


class GaussianLikelihood:
    """likelihood(f): adds the observation noise to the latent predictive (gpytorch GaussianLikelihood.__call__).
    `noise` is one float for every dataset or a tensor [B] with one noise per dataset (fitted models)."""

    def __init__(self, noise):
        self.noise = noise if torch.is_tensor(noise) else float(noise)

    def eval(self):
        return self

    def __call__(self, f):
        noise = self.noise
        if torch.is_tensor(noise):
            noise = noise.to(f.variance.device, f.variance.dtype).reshape(-1, *([1] * (f.variance.dim() - 1)))
        return _Predictive(f.mean, f.variance + noise)


class ExactGPModel:
    """Gpytorch-free stand-in for the reference's ExactGPModel (priors/fast_gp.py:13-32): constant zero mean,
    outputscale * RBF(lengthscale) kernel, exact conditioning on (train_x [B,t,F], train_y [B,t]).  Calling the model on
    test inputs [B,m,F] returns the latent predictive of each test point (batched closed form on the inputs' device)."""

    def __init__(self, train_x, train_y, likelihood, lengthscale, outputscale):
        self.train_x, self.train_y, self.likelihood = train_x, train_y, likelihood
        self.lengthscale, self.outputscale = float(lengthscale), float(outputscale)

    def eval(self):
        return self

    def to(self, device):
        self.train_x, self.train_y = self.train_x.to(device), self.train_y.to(device)
        return self

    def _k(self, a, b):
        d2 = ((a.unsqueeze(2) - b.unsqueeze(1)) / self.lengthscale).pow(2).sum(-1)
        return self.outputscale * torch.exp(-0.5 * d2)

    @torch.no_grad()
    def __call__(self, x):
        xt, yt = self.train_x.double(), self.train_y.double()
        xs = x.to(xt.device).double()
        t = xt.shape[1]
        Ktt = self._k(xt, xt) + self.likelihood.noise * torch.eye(t, dtype=xt.dtype, device=xt.device)
        Kst = self._k(xs, xt)                                   # [B,m,t]
        chol = torch.linalg.cholesky(Ktt)
        alpha = torch.cholesky_solve(yt.unsqueeze(-1), chol)    # [B,t,1]
        v = torch.cholesky_solve(Kst.transpose(1, 2), chol)     # [B,t,m]
        mean = (Kst @ alpha).squeeze(-1)
        var = self.outputscale - (Kst * v.transpose(1, 2)).sum(-1)
        return _Predictive(mean.float(), var.clamp_min(0).float())


def get_model(x, y, hyperparameters):
    """(model, likelihood) like the reference's `get_model` (priors/fast_gp.py:25-32), without gpytorch."""
    hps = _hps_to_dict(hyperparameters)
    likelihood = GaussianLikelihood(hps["noise"])
    return ExactGPModel(x, y, likelihood, hps["lengthscale"], hps["outputscale"]), likelihood


def get_model_on_device(x, y, hyperparameters, device):
    model, likelihood = get_model(x, y, hyperparameters)
    return model.to(device), likelihood


@torch.no_grad()
def evaluate(x, y, y_non_noisy, use_mse=False, hyperparameters={}, get_model_on_device=None, device=default_device,
             step_size=1, start_pos=0):
    """Exact-GP posterior baseline (reference :88-120): for each t, condition on rows < t and score row t with the
    Gaussian predictive NLL (or MSE of the predictive mean).  Returns (all_losses [n_t, B], mean losses, seconds).

    The reference builds and factors a fresh t x t model for EVERY t (T gpytorch models).  Here ONE Cholesky factor of the
    full T x T kernel matrix per dataset answers all prefixes: the leading t x t block of L is the factor of the prefix
    matrix, so with alpha = L^-1 y the prefix-t predictive of row t is
        mean_t = y_t - L_tt alpha_t ,    var_t (incl. noise) = L_tt^2 ,    NLL_t = 1/2 log(2 pi) + log L_tt + alpha_t^2 / 2 .
    The factor comes from the same fused sampler kernel that draws the prior (csrc/gp_sampler.cu).  A custom
    `get_model_on_device` (e.g. a fitted model) falls back to the reference's per-t loop on top of that callable."""
    import time
    start = time.time()
    hps = _hps_to_dict(hyperparameters if hyperparameters else None)
    if get_model_on_device is not None:
        return _evaluate_per_t(x, y, use_mse, hps, get_model_on_device, device, step_size, start_pos, start)
    dev = L.compute_device(device, _KERNEL)
    xb = x.to(dev, torch.float32).transpose(0, 1).contiguous()            # [B,T,F]
    yb = y.to(dev, torch.float32).transpose(0, 1).contiguous()            # [B,T]
    Bn, T, F = xb.shape
    ls = torch.full((Bn, F), float(hps["lengthscale"]), device=dev)
    os_ = torch.full((Bn,), float(hps["outputscale"]), device=dev)
    noise = torch.full((Bn,), float(hps["noise"]), device=dev)
    _, Lf = sample_gp(xb, torch.zeros(Bn, T, device=dev), ls, os_, noise, L.KERNEL_RBF, return_factor=True)
    alpha = torch.linalg.solve_triangular(Lf.double(), yb.double().unsqueeze(-1), upper=False).squeeze(-1)   # [B,T]
    d = torch.diagonal(Lf, dim1=1, dim2=2).double()
    if use_mse:
        per_t = (d * alpha) ** 2
    else:
        per_t = 0.5 * math.log(2 * math.pi) + torch.log(d) + 0.5 * alpha ** 2
    ts = list(range(max(start_pos, 1), T, step_size))
    all_losses = per_t[:, ts].transpose(0, 1).float()                     # [n_t, B]
    means_list = ([.0] if start_pos == 0 else []) + all_losses.mean(1).tolist()
    return all_losses.to('cpu'), torch.tensor(means_list).to('cpu'), time.time() - start


def _evaluate_per_t(x, y, use_mse, hps, get_model_on_device, device, step_size, start_pos, start):
    import time
    means_list = [.0] if start_pos == 0 else []
    all_losses = []
    for t in range(max(start_pos, 1), len(x), step_size):
        model, likelihood = get_model_on_device(x[:t].transpose(0, 1), y[:t].transpose(0, 1), hps, device)
        model.eval()
        pred = likelihood(model(x[t].unsqueeze(1)))
        means = pred.mean.squeeze()
        if use_mse:
            ls = (means - y[t].to(means.device)) ** 2
        else:
            ls = -pred.log_prob(y[t].to(means.device).unsqueeze(1))
        means_list.append(ls.mean().item())
        all_losses.append(ls.flatten().float())
    return torch.stack(all_losses).to('cpu'), torch.tensor(means_list).to('cpu'), time.time() - start
