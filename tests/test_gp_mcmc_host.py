"""Host side of the fully Bayesian GP baseline: the oracle's quadrature against the Gamma closed forms, the CPU NUTS
restatement against a Gaussian and against the quadrature posterior, the potential against scikit-learn, and the C ABI's
argument checks (which run before any CUDA call)."""
import ctypes
import math
import multiprocessing as mp

import numpy as np
import pytest
import torch

from oracle import gp_mcmc_oracle as M
from transformerscandobayesianinference_b200 import _lib as L
from transformerscandobayesianinference_b200.priors import fast_gp_mix


@pytest.mark.parametrize("conc", [(0.5, 2.0, 3.0), (1.1, 0.5, 2.0), (3.0, 1.1, 0.5)])
def test_quadrature_reproduces_the_gamma_closed_forms_without_data(conc):
    from scipy.special import digamma, polygamma
    hps = {"lengthscale_concentration": conc[0], "lengthscale_rate": 6.0, "outputscale_concentration": conc[1],
           "outputscale_rate": 0.15, "noise_concentration": conc[2], "noise_rate": 0.05}
    q = M.quadrature_posterior(torch.zeros(0, 1), torch.zeros(0), hps, n=200)   # the a = 0.5 axis spans ~70 in u
    rates = (6.0, 0.15, 0.05)
    for k in range(3):
        assert abs(q["mean"][k] - (digamma(conc[k]) - math.log(rates[k]))) <= 1e-6, (k, q)
        assert abs(q["var"][k] - polygamma(1, conc[k])) <= 1e-6, (k, q)
        assert q["edge_mass"][k] < 1e-6


def _spread_check(per_chain, target, what):
    """per_chain [chains, ...] independent estimates: their mean lies within 5 standard errors of target."""
    per_chain = np.asarray(per_chain)
    m = per_chain.mean(0)
    se = per_chain.std(0, ddof=1) / math.sqrt(len(per_chain))
    z = np.abs(m - target) / se
    print(f"{what}: mean {m} target {target} se {se} z {z}")
    assert (z <= 5).all(), (what, m, target, se)


def test_cpu_nuts_samples_a_badly_scaled_gaussian():
    scales = [0.01, 1.0, 100.0]
    jobs = [(scales, 100, 300, 11, b) for b in range(256)]
    with mp.get_context("spawn").Pool(min(16, mp.cpu_count())) as pool:
        chains = pool.map(M.gaussian_chain_job, jobs, chunksize=8)
    means = np.stack([c.mean(0) for c in chains])
    second = np.stack([(c ** 2).mean(0) for c in chains])       # E[u^2] = scale^2 at mean 0
    _spread_check(means, np.zeros(3), "means")
    _spread_check(second, np.asarray(scales) ** 2, "second moments")


def _gp_data(t, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(t + 1, 1, generator=g, dtype=torch.float64)
    y = torch.sin(5 * x[:, 0]) + 0.3 * torch.randn(t + 1, generator=g, dtype=torch.float64)
    return x, y


def test_cpu_nuts_matches_the_quadrature_posterior():
    t = 10
    x, y = _gp_data(t, 3)
    q = M.quadrature_posterior(x[:t], y[:t])
    assert (q["edge_mass"] < 1e-6).all(), q
    jobs = [(x[:t].numpy(), y[:t].numpy(), None, 2.5, 100, 300, 5, b) for b in range(256)]
    with mp.get_context("spawn").Pool(min(16, mp.cpu_count())) as pool:
        chains = pool.map(M.gp_chain_job, jobs, chunksize=8)
    _spread_check(np.stack([c.mean(0) for c in chains]), q["mean"], "E[u]")
    _spread_check(np.stack([((c - q["mean"]) ** 2).mean(0) for c in chains]), q["var"], "Var[u]")


@pytest.mark.parametrize("nu", [0.5, 1.5, 2.5])
def test_potential_matches_sklearn_and_its_gradient(nu):
    from sklearn.gaussian_process import GaussianProcessRegressor
    from sklearn.gaussian_process.kernels import ConstantKernel, Matern, WhiteKernel
    rng = np.random.default_rng(int(10 * nu))
    for F in (1, 3):
        t = int(rng.integers(5, 40))
        X = rng.random((t, F))
        y = rng.standard_normal(t)
        u = rng.normal(-0.5, 0.5, F + 2)
        th = np.exp(u)
        kernel = ConstantKernel(th[F]) * Matern(length_scale=th[:F], nu=nu) + WhiteKernel(th[F + 1])
        gpr = GaussianProcessRegressor(kernel, alpha=0.0, optimizer=None, normalize_y=False).fit(X, y)
        lml = gpr.log_marginal_likelihood(gpr.kernel_.theta)
        hps = {"nu": nu}
        U = M.potential_ref(torch.tensor(X), torch.tensor(y), torch.tensor(u), hps, nu).item()
        la, lb, oa, ob, na, nb = 3.0, 6.0, 0.5, 0.15, 1.1, 0.05
        lp = sum(a * math.log(b) - math.lgamma(a) + a * v - b * math.exp(v)
                 for a, b, v in [(la, lb, ui) for ui in u[:F]] + [(oa, ob, u[F]), (na, nb, u[F + 1])])
        assert abs(-(U + lp) - lml) <= 1e-10 * abs(lml), (U, lp, lml)
        # the closed-form numpy potential of the CPU chains against autograd
        Ur, gr = M.potential_value_and_grad_ref(torch.tensor(X), torch.tensor(y), u, hps, nu)
        Un, gn = M.potential_and_grad_np(X, y, hps, nu)(u)
        assert abs(Un - Ur) <= 1e-10 * (1 + abs(Ur))
        np.testing.assert_allclose(gn, gr, rtol=1e-8, atol=1e-8 * np.abs(gr).max())


def test_counter_rng_restatement():
    # fixed values of the hash chain (uint32 wrap-around) and the uniform's 53-bit construction
    assert M.mix32(0) == 0 and M.uniform_double(0, 0) == 0.0
    assert M.uniform_double(0xFFFFFFFF, 0xFFFFFFFF) == 1.0 - 2.0 ** -53
    r = M.Rng(1, 2, 3)
    r.key(4)
    vals = [r.uniform() for _ in range(1000)]
    assert all(0.0 <= v < 1.0 for v in vals) and abs(np.mean(vals) - 0.5) < 0.05
    r.key(4)
    assert r.uniform() == vals[0]


def test_adaptation_windows_follow_stan():
    assert M.adaptation_windows(300) == [74, 99, 149, 249, 299]
    assert M.adaptation_windows(100) == [14, 89, 99]
    assert M.adaptation_windows(10) == [9]


def _desc(T=16, F=1, ts=(4,), B=2, S=10, W=10, depth=10, hyper=(3.0, 6.0, .5, .15, 1.1, .05), n_pred=1):
    d = L.gp_mcmc_desc(B, T, F, list(ts), L.KERNEL_MATERN52, hyper, S, W, 0, depth, n_pred)
    for name in ("x", "y", "samples", "step_size", "accept", "diag"):
        setattr(d, name, 16)             # never dereferenced: the checks fail first
    return d


@pytest.mark.parametrize("kw, msg", [
    (dict(T=129, ts=(128,)), b"exceeds 128 (the t x t fp64 matrix lives in shared memory)"),
    (dict(B=0), b"empty problem"),
    (dict(ts=()), b"empty problem"),
    (dict(T=16, ts=(17,)), b"outside [1, T=16]"),
    (dict(F=33), b"F=33 exceeds 32"),
    (dict(depth=0), b"max_tree_depth=0 outside [1, 10]"),
    (dict(depth=11), b"max_tree_depth=11 outside [1, 10]"),
    (dict(S=0, W=0), b"evaluates at init, which is null"),
    (dict(n_pred=0), b"n_pred=0 outside [1, 128]"),
    (dict(n_pred=129), b"n_pred=129 outside [1, 128]"),
    (dict(S=-1), b"negative"),
    (dict(hyper=(3.0, 6.0, 0.0, .15, 1.1, .05)), b"must be positive"),
])
def test_cabi_rejects_bad_arguments_before_any_cuda_call(kw, msg):
    lib = L.load()
    d = _desc(**kw)
    assert lib.pfn_gp_mcmc(ctypes.byref(d), None) != 0
    assert msg in lib.pfn_last_error()


def test_api_raises_off_cuda():
    x, y = torch.rand(10, 3, 1), torch.randn(10, 3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        fast_gp_mix.evaluate_(x, y, y, {}, device="cpu")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        fast_gp_mix.get_mcmc_model(x[:, 0], y[:, 0], {}, "cpu", 10, 10)
    with pytest.raises(ValueError, match="limit of 128"):
        fast_gp_mix.evaluate_(torch.rand(129, 2, 1), torch.randn(129, 2), None, {}, device="cpu")


def test_mean_logdensity_restates_the_reference():
    from transformerscandobayesianinference_b200.priors import fast_gp
    mean, var = torch.tensor([[0.1], [0.5], [-0.3]]), torch.tensor([[0.2], [1.0], [0.5]])
    d = fast_gp._Predictive(mean, var)
    y = torch.tensor(0.2)
    comps = torch.distributions.Normal(mean[:, 0], var[:, 0].sqrt())
    expect = torch.logsumexp(comps.log_prob(y), 0) - math.log(3)
    assert torch.allclose(fast_gp_mix.get_mean_logdensity([d], y), expect)
    lo, hi = -1.0, 2.0
    w = comps.cdf(torch.tensor(hi)) - comps.cdf(torch.tensor(lo))
    expect = torch.logsumexp(comps.log_prob(y) - torch.log(w), 0) - math.log(3)
    assert torch.allclose(fast_gp_mix.get_mean_logdensity([d], y, (lo, hi)), expect)
