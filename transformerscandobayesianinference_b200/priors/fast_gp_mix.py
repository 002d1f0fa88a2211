"""`priors.fast_gp_mix` (reference priors/fast_gp_mix.py): a mixture-of-GPs prior.  Every dataset draws its own
hyperparameters from Gamma hyperpriors (lengthscale per input dim ~ Gamma(3, 6), outputscale ~ Gamma(.5, .15),
noise ~ Gamma(1.1, .05), rate parameterisation; reference :24-52 via botorch SingleTaskGP.pyro_sample_from_prior)
and is then sampled from a Matern-nu ARD GP (nu default 2.5) by the same fused CUDA kernel as priors.fast_gp.

The botorch/pyro model objects the reference builds per group only serve to draw those hyperparameters; here they
are drawn directly with torch.distributions.Gamma on the device (botorch 0.6.0 / pyro 1.7.0 are not installed:
the hyper-prior restatement is validated distributionally — parity unpinned, see oracle/pfn_oracle.py).

The fitted-hyperparameter baseline (`get_model`, `get_fitted_model`, `evaluate`; reference :24-55, :156-169) restates
botorch's MAP fit (SingleTaskGP + Gamma priors + fit_gpytorch_model) as csrc/gp_fit.cu: one CTA per (dataset, prefix)
problem runs the whole L-BFGS fit in fp64 and forms the predictive, all problems of a call in one launch (t <= 128).

The fully Bayesian baseline (`get_mcmc_model`, `get_mean_logdensity`, `evaluate_`; reference :171-302) integrates the
same hyperparameters out by NUTS: csrc/gp_mcmc.cu runs one chain per (dataset, prefix) problem with pyro 1.7's NUTS
defaults, on the posterior given the prefix (the reference's pyro model registers no observation site; see DESIGN §4),
and forms the predictive of row t under every sample, all chains of a call in one launch (t <= 128).
"""
import math
import random
import time

import torch
from torch import nn

from .. import _lib as L
from ..bar_distribution import BarDistribution
from ..utils import default_device
from . import fast_gp
from .fast_gp import sample_gp
from .utils import get_batch_to_dataloader, on_requested_device

MIN_INFERRED_NOISE_LEVEL = 1e-4  # botorch.models.gp_regression.MIN_INFERRED_NOISE_LEVEL (noise constraint lower bound)

_NU_TO_KERNEL = {0.5: L.KERNEL_MATERN12, 1.5: L.KERNEL_MATERN32, 2.5: L.KERNEL_MATERN52}


def sample_hyperparameters(n, num_features, hyperparameters, device):
    """Per-dataset (lengthscale [n,F], outputscale [n], noise [n]) from the Gamma hyperpriors (reference :24-52)."""
    g = torch.distributions.Gamma
    hp = hyperparameters
    one = torch.ones((), device=device)
    ls = g(one * hp.get('lengthscale_concentration', 3.0), one * hp.get('lengthscale_rate', 6.0)).sample((n, num_features))
    os_ = g(one * hp.get('outputscale_concentration', .5), one * hp.get('outputscale_rate', 0.15)).sample((n,))
    noise = g(one * hp.get('noise_concentration', 1.1), one * hp.get('noise_rate', 0.05)).sample((n,))
    return ls.float().clamp_min(1e-6), os_.float().clamp_min(1e-10), noise.float().clamp_min(MIN_INFERRED_NOISE_LEVEL)


@torch.no_grad()
def get_batch(batch_size, seq_len, num_features, device=default_device, hyperparameters=None,
              batch_size_per_gp_sample=None, num_outputs=1, fix_to_range=None, equidistant_x=False, x=None, z=None):
    """-> x [T,B,F], y [T,B], target_y [T,B] (reference :58-134).  `x` / `z`: optional caller-supplied uniform inputs
    [B,T,F] and normal draws [B,T] (e.g. pinned host memory), see priors.fast_gp.get_batch; only without fix_to_range."""
    assert num_outputs == 1
    hps = hyperparameters or {}
    dev = L.compute_device(device, fast_gp._KERNEL)
    batch_size_per_gp_sample = (batch_size_per_gp_sample or max(batch_size // 10, 1))
    assert batch_size % batch_size_per_gp_sample == 0
    kernel_type = _NU_TO_KERNEL[float(hps.get('nu', 2.5))]
    mult = 2 ** (fix_to_range is not None)
    total = batch_size * mult
    cand = batch_size_per_gp_sample * mult
    given_z = None
    if x is not None or z is not None:
        assert fix_to_range is None, "caller-supplied x / z cannot be combined with the rejection loop of fix_to_range"
    if z is not None:
        given_z = z.to(dev, torch.float32, non_blocking=True).contiguous()
    if x is not None:
        assert x.shape == (total, seq_len, num_features)
        x = x.to(dev, torch.float32, non_blocking=True).contiguous()
    elif equidistant_x:
        assert num_features == 1
        x = torch.linspace(0, 1., seq_len, device=dev).view(1, seq_len, 1).repeat(total, 1, 1)
    else:
        x = torch.rand(total, seq_len, num_features, device=dev)

    # post-processing reads y right away, so the deferred (sync-free) pivot check of sample_gp only applies to plain draws
    plain = fix_to_range is None and not hps.get('y_minmax_norm') and not hps.get('sigmoid')

    def draw(xs):
        n = xs.shape[0]
        ls, os_, noise = sample_hyperparameters(n, num_features, hps, dev)
        z = given_z if given_z is not None else torch.randn(n, seq_len, device=dev)
        s = sample_gp(xs.contiguous(), z, ls, os_, noise, kernel_type, may_defer=plain)   # [n, T]
        if hps.get('y_minmax_norm'):
            lo, hi = s.min(1, keepdim=True)[0], s.max(1, keepdim=True)[0]
            s = (s - lo) / (hi - lo)
        if hps.get('sigmoid'):
            s = s.sigmoid()
        return s

    if fix_to_range is None:
        sample = draw(x)                      # all groups in one launch: the groups are independent draws
    else:
        pieces = []
        throwaway = 0.
        for i in range(0, total, cand):
            tries = 0
            while True:
                s = draw(x[i:i + cand])
                ok = ~((s < fix_to_range[0]) | (s >= fix_to_range[1])).any(1)
                throwaway += float((~ok[:batch_size_per_gp_sample]).sum()) / batch_size_per_gp_sample
                if int(ok.sum()) >= batch_size_per_gp_sample:
                    break
                tries += 1
                if tries < 100:
                    print("Please change hyper-parameters (e.g. decrease outputscale_mean) it"
                          "seems like the range is set to tight for your hyper-parameters.")
            x[i:i + batch_size_per_gp_sample] = x[i:i + cand][ok][:batch_size_per_gp_sample]
            pieces.append(s[ok][:batch_size_per_gp_sample])
        if random.random() < .01:
            print('throwaway share', throwaway / (batch_size // batch_size_per_gp_sample))
        sample = torch.cat(pieces, 0)
        x = x.view(-1, batch_size, seq_len, num_features)[0]
    x_t, y_t = x.transpose(0, 1), sample.transpose(0, 1)
    assert x_t.shape[:2] == y_t.shape[:2]
    x_t, y_t = on_requested_device(device, x_t, y_t)
    return x_t, y_t, y_t


class DataLoader(get_batch_to_dataloader(get_batch)):
    num_outputs = 1

    @torch.no_grad()
    def validate(self, model, step_size=1, start_pos=0):
        """MSE of the bar-distribution mean at the first query row for every eval position (reference :140-153)."""
        if isinstance(model.criterion, BarDistribution):
            (x, y), target_y = self.gbm(**self.get_batch_kwargs, fuse_x_y=self.fuse_x_y)
            dev = next(model.parameters()).device
            x, y, target_y = x.to(dev), y.to(dev), target_y.to(dev)
            model.eval()
            losses = []
            mse = nn.MSELoss()
            for eval_pos in range(start_pos, len(x), step_size):
                logits = model((x, y), single_eval_pos=eval_pos)
                means = model.criterion.mean(logits)
                losses.append(mse(means[0], target_y[eval_pos]))
            model.train()
            return torch.stack(losses)
        return 123.


# ----------------------------------------------------------------------------------------------------------------------
# fitted-hyperparameter GP baseline (reference :24-55 get_model(sample=False), :156-169 get_fitted_model / evaluate)
# ----------------------------------------------------------------------------------------------------------------------
MAX_FIT_T = L.GP_FIT_MAX_T
FIT_FTOL, FIT_GTOL, FIT_MAX_ITER = 2.220446049250313e-09, 1e-5, 15000     # scipy L-BFGS-B defaults (fit_gpytorch_model)
_STATUS_NAMES = {L.GP_FIT_CONVERGED: "converged", L.GP_FIT_MAX_ITER: "iteration cap",
                 L.GP_FIT_LINE_SEARCH: "line-search failure", L.GP_FIT_NOT_PD: "not positive definite"}


def _fit_settings(hyperparameters):
    """(kernel type, Gamma prior parameters, initial noise) from the same keys and defaults as sample_hyperparameters.
    The initial noise is the noise prior's mode (reference :27-35); below the bound it is clamped to the bound."""
    hp = hyperparameters or {}
    prior = tuple(float(hp.get(k, v)) for k, v in (
        ('lengthscale_concentration', 3.0), ('lengthscale_rate', 6.0), ('outputscale_concentration', .5),
        ('outputscale_rate', 0.15), ('noise_concentration', 1.1), ('noise_rate', 0.05)))
    noise_init = max((prior[4] - 1.0) / prior[5], MIN_INFERRED_NOISE_LEVEL)
    return _NU_TO_KERNEL[float(hp.get('nu', 2.5))], prior, noise_init


def _check_fit_args(hyperparameters):
    hp = hyperparameters or {}
    assert not (hp.get('sigmoid', False)) and not (hp.get('y_minmax_norm', False)), \
        "Sigmoid and y_minmax_norm can only be used to sample models..."


_FIT_KERNEL = "priors.fast_gp_mix fits with the sm_90a GP-fit kernel"


def default_theta(n, num_features, hyperparameters, device):
    """The fit's starting point per problem: rho = 0 (lengthscales and outputscale softplus(0) = ln 2), noise at the
    noise prior's mode, constant mean 0.  Layout of theta: (rho_1..F, rho_outputscale, noise, mean)."""
    theta = torch.zeros(n, num_features + 3, dtype=torch.float64, device=device)
    theta[:, num_features + 1] = _fit_settings(hyperparameters)[2]
    return theta


@torch.no_grad()
def fit_map(x, y, ts, hyperparameters=None, theta0=None, max_iter=FIT_MAX_ITER, grad=False):
    """One pfn_gp_fit launch over every (prefix t in ts, dataset b): x [B,T,F], y [B,T] on a CUDA device.
    Returns a dict of tensors with leading dims [len(ts), B]: theta [.., F+3], f, mean / var (latent predictive of row t,
    NaN where t == T), iters, nevals, status (L.GP_FIT_*), and grad [.., F+3] when asked.  theta0 [len(ts), B, F+3]
    replaces the default start; max_iter = 0 only evaluates f, its gradient and the predictive at the start."""
    Bn, T, F = x.shape
    if T > MAX_FIT_T:
        raise ValueError(f"the GP fit keeps the t x t matrix in shared memory: T={T} exceeds the limit of {MAX_FIT_T}")
    kt, prior, noise_init = _fit_settings(hyperparameters)
    dev = x.device
    P = len(ts) * Bn
    f64 = dict(dtype=torch.float64, device=dev)
    i32 = dict(dtype=torch.int32, device=dev)
    out = {"theta": torch.empty(P, F + 3, **f64), "f": torch.empty(P, **f64), "mean": torch.empty(P, **f64),
           "var": torch.empty(P, **f64), "iters": torch.empty(P, **i32), "nevals": torch.empty(P, **i32),
           "status": torch.empty(P, **i32)}
    if grad:
        out["grad"] = torch.empty(P, F + 3, **f64)
    desc = L.gp_fit_desc(Bn, T, F, ts, kt, prior, MIN_INFERRED_NOISE_LEVEL, noise_init, max_iter, FIT_MAX_ITER,
                         FIT_FTOL, FIT_GTOL)
    th0 = None if theta0 is None else theta0.to(dev, torch.float64).reshape(P, F + 3).contiguous()
    L.gp_fit(x.to(torch.float32).contiguous(), y.to(torch.float32).contiguous(), desc, out["theta"], out["f"],
             out["iters"], out["nevals"], out["status"], theta0=th0, grad=out.get("grad"), mean=out["mean"],
             var=out["var"])
    return {k: v.view(len(ts), Bn, *v.shape[1:]) for k, v in out.items()}


class FittedGP:
    """Gpytorch-free stand-in for the reference's SingleTaskGP (constant mean, outputscale * Matern-nu ARD kernel, Gamma
    priors) on train_x [B,t,F], train_y [B,t], at the parameters `theta` [B, F+3] (raw: rho_1..F, rho_s, noise, mean).
    Calling it on test inputs [B,m,F] returns the latent predictive of each test point, formed by the same kernel that
    fits (one max_iter = 0 launch per test point), so it agrees bitwise with the predictive `evaluate` forms."""

    def __init__(self, train_x, train_y, theta, hyperparameters, likelihood, fit=None):
        self.train_x, self.train_y, self.theta = train_x, train_y, theta
        self.hyperparameters, self.likelihood = hyperparameters, likelihood
        F = train_x.shape[-1]
        self.lengthscale = torch.nn.functional.softplus(theta[:, :F])
        self.outputscale = torch.nn.functional.softplus(theta[:, F])
        self.noise = theta[:, F + 1]
        self.mean_constant = theta[:, F + 2]
        fit = fit or {}
        self.f, self.status = fit.get("f"), fit.get("status")
        self.iters, self.nevals = fit.get("iters"), fit.get("nevals")

    def eval(self):
        return self

    def train(self, mode=True):
        return self

    def to(self, device):
        self.train_x, self.train_y, self.theta = self.train_x.to(device), self.train_y.to(device), self.theta.to(device)
        return self

    @torch.no_grad()
    def __call__(self, x):
        dev = self.train_x.device
        if dev.type != 'cuda':
            raise RuntimeError("FittedGP predicts with the sm_90a GP-fit kernel; move the model to a CUDA device "
                               "(there is no CPU fallback)")
        Bn, t, F = self.train_x.shape
        xs = x.to(dev, torch.float32)
        ycat = torch.cat([self.train_y.to(torch.float32), torch.zeros(Bn, 1, device=dev)], 1).contiguous()
        means, variances = [], []
        for j in range(xs.shape[1]):
            xcat = torch.cat([self.train_x.to(torch.float32), xs[:, j:j + 1]], 1).contiguous()
            r = fit_map(xcat, ycat, [t], self.hyperparameters, theta0=self.theta.unsqueeze(0), max_iter=0)
            means.append(r["mean"][0])
            variances.append(r["var"][0])
        return fast_gp._Predictive(torch.stack(means, 1), torch.stack(variances, 1))


def get_model(x, y, hyperparameters, sample=False):
    """(model, likelihood) at the fit's starting point (reference :24-55 with sample=False).  x [B,t,F], y [B,t]."""
    if sample:
        raise NotImplementedError("priors.fast_gp_mix.get_model(sample=True): models drawn from the hyper-priors are "
                                  "sampled inside get_batch (sample_hyperparameters); use get_batch")
    _check_fit_args(hyperparameters)
    theta = default_theta(x.shape[0], x.shape[-1], hyperparameters, x.device)
    F = x.shape[-1]
    likelihood = fast_gp.GaussianLikelihood(theta[:, F + 1])
    return FittedGP(x, y, theta, hyperparameters, likelihood), likelihood


@torch.no_grad()
def get_fitted_model(x, y, hyperparameters, device):
    """MAP-fitted (model, likelihood) on x [B,t,F], y [B,t] (reference :156-166): one pfn_gp_fit launch for all B.
    The model exposes the fitted lengthscale / outputscale / noise / mean_constant and f / status / iters per dataset."""
    _check_fit_args(hyperparameters)
    dev = L.cuda_device(device, _FIT_KERNEL)
    xb, yb = x.to(dev, torch.float32).contiguous(), y.to(dev, torch.float32).contiguous()
    r = fit_map(xb, yb, [xb.shape[1]], hyperparameters)
    r = {k: v[0] for k, v in r.items()}
    F = xb.shape[-1]
    likelihood = fast_gp.GaussianLikelihood(r["theta"][:, F + 1])
    return FittedGP(xb, yb, r["theta"], hyperparameters, likelihood, fit=r), likelihood


def _report_unconverged(status):
    bad = status != L.GP_FIT_CONVERGED
    n_bad = int(bad.sum())
    if n_bad:
        parts = ", ".join(f"{name}: {int((status == code).sum())}" for code, name in _STATUS_NAMES.items()
                          if code != L.GP_FIT_CONVERGED and int((status == code).sum()))
        print(f"fast_gp_mix.evaluate: {n_bad} of {status.numel()} GP fits did not converge ({parts})")


@torch.no_grad()
def evaluate(x, y, y_non_noisy, use_mse=False, hyperparameters={}, get_model_on_device=None, device=default_device,
             step_size=1, start_pos=0):
    """Fitted-GP baseline (reference :169 = fast_gp.evaluate with get_fitted_model): for each t, fit on rows < t and score
    row t with the Gaussian predictive NLL (or the squared error of the predictive mean).  Returns
    (all_losses [n_t, B], mean losses with a leading 0 when start_pos == 0, seconds), like fast_gp.evaluate.

    Every (prefix, dataset) fit runs in ONE launch.  The losses are formed from the kernel's predictive by the same
    expressions as fast_gp's per-t loop, so `fast_gp.evaluate(..., get_model_on_device=get_fitted_model)` returns the
    same losses bit for bit.  A caller-supplied `get_model_on_device` is handed to fast_gp.evaluate."""
    if get_model_on_device is not None:
        return fast_gp.evaluate(x, y, y_non_noisy, use_mse=use_mse, hyperparameters=hyperparameters,
                                get_model_on_device=get_model_on_device, device=device, step_size=step_size,
                                start_pos=start_pos)
    start = time.time()
    _check_fit_args(hyperparameters)
    T = len(x)
    if T > MAX_FIT_T:
        raise ValueError(f"fast_gp_mix.evaluate keeps the t x t matrix of every fit in shared memory: T={T} exceeds "
                         f"the limit of {MAX_FIT_T}")
    dev = L.cuda_device(device, _FIT_KERNEL)
    ts = list(range(max(start_pos, 1), T, step_size))
    means_list = [.0] if start_pos == 0 else []
    if not ts:
        return torch.zeros(0, x.shape[1]), torch.tensor(means_list), time.time() - start
    xb = x.to(dev, torch.float32).transpose(0, 1).contiguous()
    yb = y.to(dev, torch.float32).transpose(0, 1).contiguous()
    r = fit_map(xb, yb, ts, hyperparameters)
    _report_unconverged(r["status"])
    F = xb.shape[-1]
    noise = r["theta"][..., F + 1]
    pred = fast_gp._Predictive(r["mean"].unsqueeze(-1), (r["var"] + noise).unsqueeze(-1))
    y_t = y[ts].to(dev)
    if use_mse:
        losses = (pred.mean.squeeze(-1) - y_t) ** 2
    else:
        losses = -pred.log_prob(y_t.unsqueeze(-1))
    means_list += losses.mean(1).tolist()
    return losses.float().to('cpu'), torch.tensor(means_list).to('cpu'), time.time() - start


# ----------------------------------------------------------------------------------------------------------------------
# fully Bayesian GP baseline (reference :171-268 get_mcmc_model / get_mean_logdensity / evaluate_, :274-302 __main__)
# ----------------------------------------------------------------------------------------------------------------------
MCMC_NUM_SAMPLES, MCMC_WARMUP_STEPS, MCMC_MAX_TREE_DEPTH = 100, 300, L.GP_MCMC_MAX_DEPTH


@torch.no_grad()
def sample_posterior(x, y, ts, hyperparameters=None, num_samples=MCMC_NUM_SAMPLES, warmup_steps=MCMC_WARMUP_STEPS,
                     seed=None, init=None, max_tree_depth=MCMC_MAX_TREE_DEPTH, trace=False, n_pred=1):
    """One pfn_gp_mcmc launch: a NUTS chain for every (prefix t in ts, dataset b), x [B,T,F], y [B,T] on a CUDA device.
    Returns a dict of tensors with leading dims [len(ts), B]: samples [.., S', F+2] (lengthscales, outputscale, noise),
    log_samples (the same as u = log theta), mean / var [.., S'] (latent predictive of row t per sample, NaN where
    t == T; [.., S', n_pred] for rows t .. t + n_pred - 1 when n_pred > 1), potential and grad [.., F+2] (U and dU/du at the last state), step_size, accept (mean acceptance statistic
    of the sampling phase), diag [.., 6] int32 (columns L.GP_MCMC_DIAG_NAMES), and "seed".  S' = max(num_samples, 1).
    init [len(ts), B, F+2] gives the starting u; num_samples = warmup_steps = 0 then only evaluates U, its gradient and
    the predictive at init.  num_samples = 0 with warmup_steps > 0 runs the warmup only: the one sample is the state the
    warmup ended in (samples = exp(u), log_samples = u), the predictive is formed at it and accept is NaN.  A chain
    without a finite starting point is not run: its samples and predictive are NaN.
    trace=True adds "trace" [.., W+S, F+4]: per iteration u, the step size used and the tree
    depth."""
    Bn, T, F = x.shape
    if T > MAX_FIT_T:
        raise ValueError(f"the GP sampler keeps the t x t matrix in shared memory: T={T} exceeds the limit of {MAX_FIT_T}")
    dev = L.cuda_device(x.device, _FIT_KERNEL)
    kt, prior, _ = _fit_settings(hyperparameters)
    seed = L.draw_seed(seed)
    P, So = len(ts) * Bn, max(int(num_samples), 1)
    f64 = dict(dtype=torch.float64, device=dev)
    out = L.mcmc_outputs(P, F + 2, num_samples, warmup_steps, trace, dev)
    out.update(log_samples=torch.empty(P, So, F + 2, **f64), mean=torch.empty(P, So, n_pred, **f64),
               var=torch.empty(P, So, n_pred, **f64))
    desc = L.gp_mcmc_desc(Bn, T, F, ts, kt, prior, num_samples, warmup_steps, seed, max_tree_depth, n_pred)
    u0 = None if init is None else init.to(dev, torch.float64).reshape(P, F + 2).contiguous()
    L.gp_mcmc(x.to(dev, torch.float32).contiguous(), y.to(dev, torch.float32).contiguous(), desc, out["samples"],
              out["step_size"], out["accept"], out["diag"], init=u0, log_samples=out["log_samples"], mean=out["mean"],
              var=out["var"], potential=out["potential"], grad=out["grad"], trace=out.get("trace"))
    if n_pred == 1:
        out["mean"], out["var"] = out["mean"][..., 0], out["var"][..., 0]
    r = {k: v.view(len(ts), Bn, *v.shape[1:]) for k, v in out.items()}
    r["seed"] = seed
    return r


class _SampleNoiseLikelihood:
    """likelihood(f) of a sample-batched predictive: adds every sample's own noise (gpytorch GaussianLikelihood on the
    batch of GPs pyro_load_from_samples builds).  noise [..., S] against mean / variance [..., S, m]."""

    def __init__(self, noise):
        self.noise = noise

    def eval(self):
        return self

    def __call__(self, f):
        return fast_gp._Predictive(f.mean, f.variance + self.noise.to(f.variance.dtype).unsqueeze(-1))


class MCMCGP:
    """The batch of S GPs the reference loads from the NUTS samples (pyro_load_from_samples), on train_x [B,t,F],
    train_y [B,t].  Calling it on test inputs [m,F] (or [B,m,F]) returns the latent predictive of every sample,
    mean / variance [S,m] (or [B,S,m]), formed by the sampling kernel in evaluate-only mode at the exact sampled u (one
    launch, one factorisation per sample for all m points), so it agrees bitwise with the predictive `evaluate_` forms."""

    def __init__(self, train_x, train_y, r, hyperparameters, batched):
        self.train_x, self.train_y, self.hyperparameters, self.batched = train_x, train_y, hyperparameters, batched
        F = train_x.shape[-1]
        self.samples, self.log_samples = r["samples"], r["log_samples"]          # [B, S, F+2]
        self.lengthscale = self.samples[..., :F]
        self.outputscale = self.samples[..., F]
        self.noise = self.samples[..., F + 1]
        self.step_size, self.accept, self.diag, self.seed = r["step_size"], r["accept"], r["diag"], r["seed"]

    def eval(self):
        return self

    def train(self, mode=True):
        return self

    @torch.no_grad()
    def __call__(self, x):
        Bn, t, F = self.train_x.shape
        S = self.samples.shape[1]
        xs = x.to(self.train_x.device, torch.float32).reshape(Bn, -1, F)
        m = xs.shape[1]
        if t + m > MAX_FIT_T:
            raise ValueError(f"the GP sampler keeps the data and the test points in shared memory: t + m = {t + m} "
                             f"exceeds the limit of {MAX_FIT_T}")
        xcat = torch.cat([self.train_x.to(torch.float32), xs], 1).repeat_interleave(S, 0).contiguous()   # q = b * S + s
        ycat = torch.cat([self.train_y.to(torch.float32), torch.zeros(Bn, m, device=xs.device)], 1)
        init = self.log_samples.reshape(1, Bn * S, F + 2)
        r = sample_posterior(xcat, ycat.repeat_interleave(S, 0).contiguous(), [t], self.hyperparameters, 0, 0, seed=0,
                             init=init, n_pred=m)
        mean, var = r["mean"][0, :, 0].reshape(Bn, S, m), r["var"][0, :, 0].reshape(Bn, S, m)
        if not self.batched:
            mean, var = mean[0], var[0]
        return fast_gp._Predictive(mean, var)


@torch.no_grad()
def get_mcmc_model(x, y, hyperparameters, device, num_samples, warmup_steps, seed=None):
    """(model, likelihood) after one NUTS chain per dataset (reference :171-196): x [t,F] and y [t] as the reference
    passes them, or a batch x [B,t,F], y [B,t].  The model is the batch of GPs at the S samples (MCMCGP), the
    likelihood adds each sample's noise."""
    _check_fit_args(hyperparameters)
    dev = L.cuda_device(device, _FIT_KERNEL)
    batched = x.dim() == 3
    xb = (x if batched else x.unsqueeze(0)).to(dev, torch.float32).contiguous()
    yb = (y if batched else y.unsqueeze(0)).to(dev, torch.float32).reshape(xb.shape[0], xb.shape[1]).contiguous()
    r = sample_posterior(xb, yb, [xb.shape[1]], hyperparameters, num_samples, warmup_steps, seed=seed)
    r = {k: (v[0] if torch.is_tensor(v) else v) for k, v in r.items()}
    model = MCMCGP(xb, yb, r, hyperparameters, batched)
    noise = model.noise if batched else model.noise[0]
    return model, _SampleNoiseLikelihood(noise)


def _mixture_logdensity(mean, var, y, full_range=None):
    """log of the equal-weight Gaussian mixture over the last dim of mean / var at y (broadcast over the rest), each
    component renormalised to full_range when given (reference :203-217)."""
    dist = torch.distributions.Normal(mean, var.sqrt())
    logprobs = dist.log_prob(y.unsqueeze(-1))
    if full_range is not None:
        used_weight = 1. - (dist.cdf(torch.tensor(full_range[0])) + (1. - dist.cdf(torch.tensor(full_range[1]))))
        if torch.isinf(-torch.log(used_weight)).any() or torch.isinf(torch.log(used_weight)).any():
            print('factor is inf', -torch.log(used_weight))
        logprobs = logprobs - torch.log(used_weight)
    return torch.logsumexp(logprobs, -1) - math.log(logprobs.shape[-1])


def get_mean_logdensity(dists, x, full_range=None):
    """Log density at x of the equal-weight mixture of the predictives in `dists` (reference :203-217)."""
    means = torch.cat([d.mean.squeeze() for d in dists], 0)
    vars = torch.cat([d.variance.squeeze() for d in dists], 0)
    assert len(means.shape) == 1 and len(vars.shape) == 1
    return _mixture_logdensity(means, vars, torch.as_tensor(x, dtype=means.dtype, device=means.device), full_range)


def _report_mcmc(diag, samples):
    n_dead = int(torch.isnan(samples[..., 0, 0]).sum())
    if n_dead:
        print(f"fast_gp_mix.evaluate_: {n_dead} chains found no finite starting point and were not run (NaN losses)")
    n_div, n_depth = L.mcmc_trouble(diag)
    if n_div or n_depth:
        print(f"fast_gp_mix.evaluate_: {diag.shape[0] * diag.shape[1]} chains: {n_div} sampling iterations diverged, "
              f"{n_depth} iterations (warmup included) hit the tree-depth cap")


@torch.no_grad()
def evaluate_(x, y, y_non_noisy, hyperparameters=None, device=default_device, num_samples=MCMC_NUM_SAMPLES,
              warmup_steps=MCMC_WARMUP_STEPS, full_range=None, min_seq_len=0, use_likelihood=False, seed=None):
    """Fully Bayesian GP baseline (reference :220-268): for each t >= max(min_seq_len, 1) and dataset b, NUTS on rows < t
    of x [T,B,F], y [T,B], then minus the log density of y[t, b] under the mixture of the S sample predictives (with each
    sample's noise when use_likelihood).  Returns (losses_after_t [n_t (+1)], seconds, all_losses) like the reference:
    the per-t mean losses with a leading 0 when min_seq_len == 0, and the per-(t, b) losses as lists.

    Every (t, b) chain runs in ONE launch; `seed` (default: drawn from torch's CPU generator) fixes all chains, so the
    result equals a per-t loop over `get_mcmc_model(x[:t].transpose(0, 1), ...)` with the same seed."""
    start_time = time.time()
    hps = hyperparameters or {}
    _check_fit_args(hps)
    T = len(x)
    if T > MAX_FIT_T:
        raise ValueError(f"fast_gp_mix.evaluate_ keeps the t x t matrix of every chain in shared memory: T={T} exceeds "
                         f"the limit of {MAX_FIT_T}")
    dev = L.cuda_device(device, _FIT_KERNEL)
    losses_after_t = [.0] if min_seq_len == 0 else []
    ts = list(range(max(min_seq_len, 1), T))
    if not ts:
        return torch.tensor(losses_after_t), time.time() - start_time, []
    xb = x.to(dev, torch.float32).transpose(0, 1).contiguous()
    yb = y.to(dev, torch.float32).transpose(0, 1).contiguous()
    r = sample_posterior(xb, yb, ts, hps, num_samples, warmup_steps, seed=seed)
    _report_mcmc(r["diag"], r["samples"])
    F = xb.shape[-1]
    var = r["var"] + r["samples"][..., F + 1] if use_likelihood else r["var"]
    losses = -_mixture_logdensity(r["mean"], var, y[ts].to(dev, torch.float64), full_range)     # [n_t, B]
    all_losses = losses.tolist()
    losses_after_t += losses.mean(1).tolist()
    return torch.tensor(losses_after_t), time.time() - start_time, all_losses


if __name__ == '__main__':
    import argparse

    parser = argparse.ArgumentParser()
    parser.add_argument('--batch_size', type=int)
    parser.add_argument('--seq_len', type=int)
    parser.add_argument('--min_seq_len', type=int, default=0)
    parser.add_argument('--warmup_steps', type=int)
    parser.add_argument('--num_samples', type=int)
    parser.add_argument('--min_y', type=int)
    parser.add_argument('--max_y', type=int)
    parser.add_argument('--dim', type=int, default=1)
    parser.add_argument('--use_likelihood', default=True, type=bool)
    parser.add_argument('--device', default='cuda')
    parser.add_argument('--outputscale_concentraion', default=2., type=float)
    parser.add_argument('--noise_concentration', default=1.1, type=float)
    parser.add_argument('--noise_rate', default=.05, type=float)

    args = parser.parse_args()

    print('min_y:', args.min_y)
    full_range = (None if args.min_y is None else (args.min_y, args.max_y))

    # fast_computations only switches gpytorch's approximate solves, which this exact fp64 path does not have
    hps = {'outputscale_concentration': args.outputscale_concentraion, 'noise_concentration': args.noise_concentration,
           'noise_rate': args.noise_rate, 'fast_computations': (False, False, False)}
    x, y, _ = get_batch(args.batch_size, args.seq_len, args.dim, device=args.device, fix_to_range=full_range,
                        hyperparameters=hps)
    print('RESULT:', evaluate_(x, y, y, device=args.device, warmup_steps=args.warmup_steps,
                               num_samples=args.num_samples, full_range=full_range, min_seq_len=args.min_seq_len,
                               hyperparameters=hps, use_likelihood=args.use_likelihood))
