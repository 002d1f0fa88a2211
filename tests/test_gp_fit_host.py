"""Fitted-hyperparameter GP baseline, host side (no GPU): the oracle's marginal likelihood against scikit-learn, the C-ABI
argument checks of pfn_gp_fit (made before any CUDA call) and the Python API's argument handling."""
import ctypes
import math
import sys

import numpy as np
import pytest
import torch

from oracle import gp_fit_oracle as G
from transformerscandobayesianinference_b200 import _lib as L
from transformerscandobayesianinference_b200.priors import fast_gp_mix


def _softplus(v):
    return math.log1p(math.exp(v))


def _sigmoid(v):
    return 1.0 / (1.0 + math.exp(-v))


@pytest.mark.parametrize("nu", [0.5, 1.5, 2.5])
@pytest.mark.parametrize("F", [1, 3])
def test_marginal_likelihood_matches_sklearn(nu, F):
    from sklearn.gaussian_process import GaussianProcessRegressor
    from sklearn.gaussian_process.kernels import ConstantKernel, Matern, WhiteKernel
    rng = np.random.default_rng(100 * F + int(10 * nu))
    for _ in range(4):
        t = int(rng.integers(5, 40))
        X = rng.random((t, F))
        y = rng.normal(size=t)
        params = np.concatenate([rng.normal(-1.0, 0.7, size=F + 1), [rng.uniform(0.01, 0.5), 0.0]])
        ls = [_softplus(v) for v in params[:F]]
        s, noise = _softplus(params[F]), params[F + 1]
        kernel = ConstantKernel(s) * Matern(length_scale=np.array(ls), nu=nu) + WhiteKernel(noise)
        gpr = GaussianProcessRegressor(kernel, alpha=0.0, optimizer=None, normalize_y=False).fit(X, y)
        lml, lml_grad = gpr.log_marginal_likelihood(gpr.kernel_.theta, eval_gradient=True)   # d/d log(s, ls.., noise)
        p = torch.tensor(params, dtype=torch.float64, requires_grad=True)
        f = G.gp_map_objective_ref(torch.tensor(X), torch.tensor(y), p, nu=nu, priors=False)
        (g,) = torch.autograd.grad(f, p)
        assert abs(-t * f.item() - lml) <= 1e-10 * abs(lml)
        expect = np.zeros(F + 3)
        expect[F] = -lml_grad[0] / s * _sigmoid(params[F]) / t
        for d in range(F):
            expect[d] = -lml_grad[1 + d] / ls[d] * _sigmoid(params[d]) / t
        expect[F + 1] = -lml_grad[F + 1] / noise / t
        expect[F + 2] = g[F + 2].item()            # the constant mean is not a sklearn parameter (checked below)
        np.testing.assert_allclose(g.numpy(), expect, rtol=1e-8, atol=1e-8 * np.abs(expect).max())
        # d/dc log N(y | c, K) = 1^T K^-1 (y - c)
        K = gpr.kernel_(X)
        assert abs(-t * g[F + 2].item() - np.linalg.solve(K, y).sum()) <= 1e-8 * (1 + abs(np.linalg.solve(K, y).sum()))


def test_oracle_fit_reaches_a_stationary_point():
    torch.manual_seed(0)
    x = torch.rand(20, 2, dtype=torch.float64)
    y = torch.sin(6 * x[:, 0]) + 0.1 * torch.randn(20, dtype=torch.float64)
    r = G.gp_fit_ref(x, y, x_test=torch.tensor([0.5, 0.5], dtype=torch.float64))
    f0, _ = G.gp_map_value_and_grad_ref(x, y, G.gp_default_theta_ref(2))
    f, g = G.gp_map_value_and_grad_ref(x, y, r["theta"])
    # scipy stops on the relative reduction of f (ftol) as often as on the projected gradient (gtol)
    assert r["success"] and f <= f0 and G.gp_projected_grad_norm_ref(r["theta"], g, 2) <= 1e-3
    assert r["var"] > 0 and math.isfinite(r["mean"])


def _desc(T=16, F=1, ts=(4,), B=2):
    d = L.gp_fit_desc(B, T, F, list(ts), L.KERNEL_MATERN52, (3.0, 6.0, .5, .15, 1.1, .05), 1e-4, 2.0, 100, 100, 1e-9, 1e-5)
    for name in ("x", "y", "theta", "f", "iters", "nevals", "status"):
        setattr(d, name, 16)             # never dereferenced: the checks fail first
    return d


@pytest.mark.parametrize("kw, msg", [
    (dict(T=129, ts=(128,)), b"exceeds 128"),
    (dict(B=0), b"empty problem"),
    (dict(ts=()), b"empty problem"),
    (dict(T=16, ts=(17,)), b"outside [1, T=16]"),
    (dict(ts=(0,)), b"outside"),
    (dict(F=33), b"F=33 exceeds 32"),
])
def test_cabi_rejects_bad_arguments_before_any_cuda_call(kw, msg):
    lib = L.load()
    d = _desc(**kw)
    assert lib.pfn_gp_fit(ctypes.byref(d), None) != 0
    assert msg in lib.pfn_last_error()


def test_cabi_rejects_a_non_matern_kernel():
    lib = L.load()
    d = _desc()
    d.kernel_type = L.KERNEL_RBF
    assert lib.pfn_gp_fit(ctypes.byref(d), None) != 0 and b"not a Matern kernel" in lib.pfn_last_error()


def test_api_argument_handling_on_the_host():
    x, y = torch.rand(10, 3, 1), torch.randn(10, 3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        fast_gp_mix.evaluate(x, y, y, device="cpu")
    with pytest.raises(ValueError, match="limit of 128"):
        fast_gp_mix.evaluate(torch.rand(129, 2, 1), torch.randn(129, 2), None, device="cuda:0")
    with pytest.raises(AssertionError, match="Sigmoid and y_minmax_norm"):
        fast_gp_mix.evaluate(x, y, y, hyperparameters={"sigmoid": True}, device="cuda:0")
    with pytest.raises(AssertionError, match="Sigmoid and y_minmax_norm"):
        fast_gp_mix.get_model(x.transpose(0, 1), y.transpose(0, 1), {"y_minmax_norm": True})
    with pytest.raises(NotImplementedError, match="get_batch"):
        fast_gp_mix.get_model(x.transpose(0, 1), y.transpose(0, 1), {}, sample=True)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        fast_gp_mix.get_fitted_model(x.transpose(0, 1), y.transpose(0, 1), {}, "cpu")


def test_model_at_the_starting_point():
    model, likelihood = fast_gp_mix.get_model(torch.rand(3, 7, 2), torch.randn(3, 7), {})
    assert torch.allclose(model.lengthscale, torch.full((3, 2), math.log(2.0), dtype=torch.float64))
    assert torch.allclose(model.outputscale, torch.full((3,), math.log(2.0), dtype=torch.float64))
    assert torch.equal(model.noise, torch.full((3,), (1.1 - 1.0) / 0.05, dtype=torch.float64))   # the noise prior's mode
    assert torch.equal(model.mean_constant, torch.zeros(3, dtype=torch.float64))
    assert likelihood is model.likelihood
    # a noise prior whose mode lies below the bound starts at the bound
    model, _ = fast_gp_mix.get_model(torch.rand(1, 4, 1), torch.randn(1, 4), {"noise_concentration": 0.5})
    assert model.noise.item() == fast_gp_mix.MIN_INFERRED_NOISE_LEVEL


def test_likelihood_takes_a_float_or_one_noise_per_dataset():
    from transformerscandobayesianinference_b200.priors import fast_gp
    f = fast_gp._Predictive(torch.zeros(3, 1), torch.ones(3, 1))
    assert torch.equal(fast_gp.GaussianLikelihood(0.5)(f).variance, torch.full((3, 1), 1.5))
    noisy = fast_gp.GaussianLikelihood(torch.tensor([0.1, 0.2, 0.3]))(f)
    assert torch.allclose(noisy.variance, torch.tensor([[1.1], [1.2], [1.3]]))


def test_dropin_exposes_the_fitted_baseline():
    import transformerscandobayesianinference_b200 as pfn
    saved = {k: sys.modules.get(k) for k in list(sys.modules) if k.split(".")[0] in pfn._DROPIN_MODULES}
    try:
        pfn.install_dropin()
        mod = sys.modules["priors.fast_gp_mix"]
        assert mod.evaluate is fast_gp_mix.evaluate and mod.get_fitted_model is fast_gp_mix.get_fitted_model
        assert mod.get_model is fast_gp_mix.get_model
    finally:
        for k in [k for k in list(sys.modules) if k.split(".")[0] in pfn._DROPIN_MODULES]:
            del sys.modules[k]
        sys.modules.update({k: v for k, v in saved.items() if v is not None})
