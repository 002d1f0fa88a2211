"""CPU oracle of the fitted-hyperparameter GP baseline — TEST INFRASTRUCTURE ONLY (like oracle/pfn_oracle.py: plain
torch / scipy, sharing no code with the CUDA engine; only tests/ and tools/ import it).

Restates reference priors/fast_gp_mix.py:24-55 (get_model, sample=False), :156-169 (get_fitted_model, evaluate) and
priors/fast_gp.py:88-120 (the per-t evaluate loop) in gpytorch 1.5 / botorch 0.6 terms.  PARITY UNPINNED: neither library
is installed, so the exact marginal likelihood is pinned against scikit-learn's GaussianProcessRegressor instead
(tests/test_gp_fit_host.py) and the optimiser is scipy's L-BFGS-B, the one fit_gpytorch_model drives.
"""
import math

import torch

GP_FIT_NOISE_LB = 1e-4                  # botorch MIN_INFERRED_NOISE_LEVEL, GreaterThan(..., transform=None)


def _gp_fit_priors(hps):
    hp = hps or {}
    return tuple(float(hp.get(k, v)) for k, v in (
        ('lengthscale_concentration', 3.0), ('lengthscale_rate', 6.0), ('outputscale_concentration', .5),
        ('outputscale_rate', 0.15), ('noise_concentration', 1.1), ('noise_rate', 0.05)))


def _gamma_logpdf(v, a, b):
    return a * math.log(b) - math.lgamma(a) + (a - 1.0) * torch.log(v) - b * v


def gp_matern_ref(xa, xb, ls, nu):
    """Matern-nu ARD correlation k(xa, xb) [n, m] (gpytorch MaternKernel; r = 0 pairs have k = 1 and no gradient)."""
    d2 = (((xa.unsqueeze(1) - xb.unsqueeze(0)) / ls) ** 2).sum(-1)
    r = torch.where(d2 > 0, d2.clamp_min(1e-300).sqrt(), torch.zeros_like(d2))
    a = math.sqrt(2 * nu) * r
    if nu == 0.5:
        return torch.exp(-a)
    if nu == 1.5:
        return (1 + a) * torch.exp(-a)
    return (1 + a + 5.0 / 3.0 * d2) * torch.exp(-a)


def gp_map_objective_ref(x, y, params, hps=None, nu=2.5, priors=True):
    """f(theta) = -(1/t) [log N(y | c 1, K) + log-priors] for ONE problem: x [t,F], y [t], params [F+3] =
    (rho_1..F, rho_outputscale, noise, mean); lengthscale / outputscale = softplus(rho), noise used untransformed.
    fp64 torch; differentiate with autograd.  priors=False leaves the exact marginal likelihood alone."""
    t, F = x.shape
    ls = torch.nn.functional.softplus(params[:F])
    s = torch.nn.functional.softplus(params[F])
    noise, c = params[F + 1], params[F + 2]
    K = s * gp_matern_ref(x, x, ls, nu) + noise * torch.eye(t, dtype=x.dtype)
    Lc = torch.linalg.cholesky(K)
    resid = (y - c).unsqueeze(-1)
    alpha = torch.cholesky_solve(resid, Lc)
    logn = -0.5 * (resid * alpha).sum() - torch.log(torch.diagonal(Lc)).sum() - 0.5 * t * math.log(2 * math.pi)
    if priors:
        la, lb, oa, ob, na, nb = _gp_fit_priors(hps)
        logn = logn + _gamma_logpdf(ls, la, lb).sum() + _gamma_logpdf(s, oa, ob) + _gamma_logpdf(noise, na, nb)
    return -logn / t


def gp_map_value_and_grad_ref(x, y, params, hps=None, nu=2.5):
    """(f, grad) as float64 numpy values; f = +inf (and a zero gradient) where K is not positive definite."""
    import numpy as np
    p = torch.as_tensor(np.asarray(params, dtype=np.float64)).clone().requires_grad_(True)
    try:
        f = gp_map_objective_ref(x, y, p, hps, nu)
    except torch.linalg.LinAlgError:
        return float("inf"), np.zeros(p.numel())
    (g,) = torch.autograd.grad(f, p)
    return float(f.detach()), g.numpy()


def gp_default_theta_ref(F, hps=None):
    """Starting point of the reference fit: raw lengthscale / outputscale 0 (softplus(0) = ln 2), noise at the noise
    prior's mode (GreaterThan initial_value, reference :27-35; clamped to the bound), constant mean 0."""
    na, nb = _gp_fit_priors(hps)[4:]
    th = [0.0] * (F + 3)
    th[F + 1] = max((na - 1.0) / nb, GP_FIT_NOISE_LB)
    return th


def gp_fit_ref(x, y, hps=None, nu=2.5, x_test=None, theta0=None):
    """scipy L-BFGS-B (fit_gpytorch_model's optimiser, scipy defaults) on ONE problem from the reference's start, then the
    latent predictive at x_test [F]: mean = c + k*^T K^-1 (y - c), var = s - k*^T K^-1 k*.  x [t,F], y [t] fp64."""
    import numpy as np
    from scipy.optimize import minimize
    t, F = x.shape
    th0 = np.asarray(gp_default_theta_ref(F, hps) if theta0 is None else theta0, dtype=np.float64)
    bounds = [(None, None)] * (F + 1) + [(GP_FIT_NOISE_LB, None), (None, None)]
    res = minimize(lambda p: gp_map_value_and_grad_ref(x, y, p, hps, nu), th0, jac=True, method="L-BFGS-B",
                   bounds=bounds)
    out = {"theta": res.x, "f": float(res.fun), "nit": int(res.nit), "nfev": int(res.nfev), "success": bool(res.success)}
    if x_test is not None:
        p = torch.as_tensor(res.x)
        ls, s = torch.nn.functional.softplus(p[:F]), torch.nn.functional.softplus(p[F])
        noise, c = p[F + 1], p[F + 2]
        K = s * gp_matern_ref(x, x, ls, nu) + noise * torch.eye(t, dtype=x.dtype)
        ks = s * gp_matern_ref(x, x_test.reshape(1, F), ls, nu)[:, 0]
        sol = torch.linalg.solve(K, torch.stack([y - c, ks], -1))
        out["mean"] = float(c + ks @ sol[:, 0])
        out["var"] = float(s - ks @ sol[:, 1])
    return out


def gp_projected_grad_norm_ref(theta, grad, F):
    """inf-norm of L-BFGS-B's projected gradient (the noise is bounded below by GP_FIT_NOISE_LB)."""
    g = [float(v) for v in grad]
    if g[F + 1] > 0:
        g[F + 1] = min(float(theta[F + 1]) - GP_FIT_NOISE_LB, g[F + 1])
    return max(abs(v) for v in g)


def gp_fit_ref_job(job):
    """gp_fit_ref((x, y, x_test)) on one thread: the unit of work of a process pool over many problems."""
    torch.set_num_threads(1)
    x, y, x_test = job
    return gp_fit_ref(x, y, x_test=x_test)
