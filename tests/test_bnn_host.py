"""Host side of the Bayesian-NN experiment (no GPU): the oracle's closed-form potential against autograd, the CPU NUTS
restatement on it against the importance-sampling posterior predictive, the reference's helper functions, the drop-in
module names and the argument checks of the two C-ABI entries."""
import ctypes
import math
import sys

import numpy as np
import pytest
import torch

from oracle import bnn_oracle as O
from oracle.gp_mcmc_oracle import nuts_chain
from transformerscandobayesianinference_b200 import _lib as L


def _data(F, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, F, generator=g, dtype=torch.float64), torch.randint(0, 2, (n,), generator=g)


@pytest.mark.parametrize("F,E,n", [(1, 1, 1), (3, 5, 2), (3, 5, 100), (8, 64, 7), (2, 7, 33)])
def test_numpy_potential_matches_autograd(F, E, n):
    x, y = _data(F, n, 100 * F + E + n)
    pot = O.potential_and_grad_np(x.numpy(), y.numpy(), F, E)
    g = torch.Generator().manual_seed(7)
    for scale in (0.1, 1.0, 3.0):
        th = torch.randn(O.dim(F, E), generator=g, dtype=torch.float64) * scale
        U_ref, g_ref = O.potential_value_and_grad_ref(x, y, th.numpy(), F, E)
        U, gr = pot(th.numpy())
        assert abs(U - U_ref) <= 1e-10 * (1 + abs(U_ref))
        assert np.abs(np.asarray(gr) - g_ref).max() <= 1e-8 * (1 + np.linalg.norm(g_ref))


def test_potential_is_the_negative_log_joint():
    F, E, n = 2, 3, 4
    x, y = _data(F, n, 3)
    th = torch.randn(O.dim(F, E), generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    W1, b1, W2, b2 = O.unpack(th, F, E)
    logits = (x @ W1.T + b1) @ W2.T + b2
    lj = torch.distributions.Normal(0., 1.).log_prob(th).sum() + torch.distributions.Categorical(logits=logits).log_prob(y).sum()
    assert abs(float(O.potential_ref(x, y, th, F, E)) + float(lj)) <= 1e-12 * (1 + abs(float(lj)))


def test_cpu_chains_agree_with_importance_sampling():
    F, E, n, m = 1, 1, 3, 4
    x, y = _data(F, n + m, 11)
    y[:n] = torch.tensor([1, 1, 0])
    ref = O.importance_predictive(x[:n], y[:n], x[n:], F, E, num_draws=1 << 19, seed=5)
    assert ref["ess"] > 1e4 and (ref["se"] < 2e-3).all(), ref
    pot = O.potential_and_grad_np(x[:n].numpy(), y[:n].numpy(), F, E)
    per_chain = []
    for b in range(6):                      # depth cap 6 (63 leapfrog steps) keeps the Python chains short; NUTS stays exact
        c = nuts_chain(pot, O.dim(F, E), 150, 100, seed=42, b=b, t=n, max_tree_depth=6)
        assert c["diag"]["div_sampling"] <= 3
        per_chain.append(O.predictive_ref(torch.as_tensor(c["samples"]), x[n:], F, E).mean(0).numpy())
    est = np.stack(per_chain)
    se = np.sqrt(est.var(0, ddof=1) / len(est) + ref["se"] ** 2)
    z = np.abs(est.mean(0) - ref["p1"]) / se
    print(f"chains {est.mean(0)} importance sampling {ref['p1']} se {se} z {z}")
    assert (z <= 5).all() and (np.abs(est.mean(0) - ref["p1"]) <= 0.05).all()


def test_prior_forward_ref_standardises_and_decides():
    F, E, T, B = 3, 5, 40, 2
    g = torch.Generator().manual_seed(0)
    w, xr, u = torch.randn(B, O.dim(F, E), generator=g), torch.randn(T, B, F, generator=g), torch.rand(T, B, generator=g)
    p0, y, xn = O.prior_forward_ref(w, xr, u, F, E)
    assert xn.mean(0).abs().max() < 1e-12 and (xn.std(0) - 1).abs().max() < 1e-5
    W1, b1, W2, b2 = O.unpack(w[1].double(), F, E)
    l = (xr[7, 1].double() @ W1.T + b1) @ W2.T + b2
    assert abs(float(torch.softmax(l, 0)[0]) - float(p0[7, 1])) < 1e-14
    assert torch.equal(y, (u.double() >= p0).double())


def test_reference_helpers():
    from transformerscandobayesianinference_b200 import mcmc_svi_transformer_on_bayesian as M
    assert M.get_default_model_spec('small') == {'nlayers': 2, 'embed': 5, 'num_features': 3, 'seq_len': 300}
    assert M.get_default_model_spec('big') == {'nlayers': 2, 'embed': 64, 'num_features': 8, 'seq_len': 300}
    assert M.get_default_model_spec('4_9_1') == {'nlayers': 1, 'embed': 9, 'num_features': 4, 'seq_len': 300}
    assert M.get_default_evaluation_points() == list(range(2, 100, 5))
    cfg = M.get_transformer_config(M.get_default_model_spec('small'))
    assert cfg['num_features'] == 3 and cfg['seq_len'] == 300 and cfg['emsize'] == 256 and cfg['num_outputs'] == 1
    obs = torch.tensor([[1., 0., 1.], [1., 1., 0.], [1., 0., 0.], [0., 0., 1.]])
    y = torch.tensor([1., 0., 1.])
    acc, nll, mse = M.evaluate_preds({'obs': obs}, y)
    means = torch.tensor([0.75, 0.25, 0.5])
    assert abs(float(acc) - 8 / 12) < 1e-7
    assert abs(float(nll) - float(torch.nn.BCELoss()(means, y))) < 1e-7
    assert abs(float(mse) - float(((means - y) ** 2).mean())) < 1e-7
    m, h = M.compute_mean_and_conf_interval([1.0, 2.0, 3.0, 4.0])
    assert m == 2.5 and abs(h - 2.0540) < 1e-3          # t_{0.975, 3} * sd / 2 = 3.1824 * 1.29099 / 2
    with pytest.raises(NotImplementedError, match="svi"):
        M.training_steps('svi', None, None, None)
    with pytest.raises(NotImplementedError, match="svgd"):
        M.training_samples('svgd', None, None, None, [2])
    model = M.BayesianModel({'num_features': 3, 'embed': 5, 'nlayers': 2})
    assert (model.num_features, model.embed) == (3, 5)


def test_install_dropin_registers_the_new_modules():
    import transformerscandobayesianinference_b200 as pfn
    saved = dict(sys.modules)
    try:
        mods = pfn.install_dropin()
        assert set(mods) == set(pfn._DROPIN_MODULES)
        import mcmc_svi_transformer_on_bayesian as M
        import priors.pyro as P
        assert M is pfn.mcmc_svi_transformer_on_bayesian and P is pfn.priors.pyro
        assert P.DataLoader.num_outputs == 1 and callable(P.get_batch)
    finally:
        for k in set(sys.modules) - set(saved):
            del sys.modules[k]


def test_generic_callable_path_runs_the_model_per_dataset():
    from transformerscandobayesianinference_b200.priors import pyro as P
    calls = []

    class Toy:
        def __call__(self, seq_len=1):
            calls.append(seq_len)
            x = torch.randn(seq_len, 2)
            return x, (x[:, 0] > 0).float()

    x, y, t = P.get_batch(8, 11, batch_size_per_gp_sample=4, model=Toy, device='cpu')
    assert x.shape == (11, 8, 2) and y.shape == (11, 8) and t is y and calls == [11] * 8
    assert x.mean(0).abs().max() < 1e-6
    with pytest.raises(AssertionError, match="divisible"):
        P.get_batch(8, 11, batch_size_per_gp_sample=3, model=Toy, device='cpu')


def test_cabi_argument_checks():
    lib = L.load()
    assert lib.pfn_bnn_prior(0, 0, 0, 10, 3, 5, None, None, None, None, None, None) != 0
    assert b"empty problem" in lib.pfn_last_error()
    assert lib.pfn_bnn_prior(0, 0, 4, 10, 8, 200, None, None, None, None, None, None) != 0
    assert b"exceeds 1024" in lib.pfn_last_error()
    assert lib.pfn_bnn_prior(0, 0, 4, 100000, 8, 4, None, None, None, None, None, None) != 0
    assert b"shared memory" in lib.pfn_last_error()
    assert lib.pfn_bnn_prior(0, 0, 4, 10, 3, 5, None, None, None, None, None, None) != 0
    assert b"null output" in lib.pfn_last_error()

    assert lib.pfn_bnn_mcmc(None, None) != 0 and b"null descriptor" in lib.pfn_last_error()
    d = L.bnn_mcmc_desc(0, 10, 5, 3, 5, 10, 10, 1)
    assert lib.pfn_bnn_mcmc(ctypes.byref(d), None) != 0 and b"empty problem" in lib.pfn_last_error()
    d = L.bnn_mcmc_desc(2, 10, 5, 8, 200, 10, 10, 1)
    assert lib.pfn_bnn_mcmc(ctypes.byref(d), None) != 0 and b"exceeds 1024" in lib.pfn_last_error()
    with pytest.raises(RuntimeError, match="exceeds 1024"):
        L.bnn_mcmc_workspace(d)
    d = L.bnn_mcmc_desc(2, 2000, 5, 3, 5, 10, 10, 1)
    assert lib.pfn_bnn_mcmc(ctypes.byref(d), None) != 0 and b"training rows exceed" in lib.pfn_last_error()
    d = L.bnn_mcmc_desc(2, 10, 5, 3, 5, 10, 10, 1)
    assert lib.pfn_bnn_mcmc(ctypes.byref(d), None) != 0 and b"null input or output" in lib.pfn_last_error()
    # the state of `small` (d = 32) fits in shared memory; `big` (d = 706) needs 78 d doubles of workspace per chain
    assert L.bnn_mcmc_workspace(L.bnn_mcmc_desc(100, 100, 200, 3, 5, 64, 64, 1)) == 0
    assert L.bnn_mcmc_workspace(L.bnn_mcmc_desc(100, 100, 200, 8, 64, 64, 64, 1)) == 78 * 706
