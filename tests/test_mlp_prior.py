"""priors.mlp (BNN tabular prior) against the UNMODIFIED reference priors/mlp.py (statistics of its batches recorded in
tests/golden/host_reference.pt by oracle/make_golden.py): same host hyper-sampler stream, same per-dataset distribution.  The vectorised all-models-at-once formulation is checked on
CPU here (no kernels involved: it is batched torch ops) and on the GPU through the public `get_batch`."""
import os
import random

import numpy as np
import pytest
import torch

from transformerscandobayesianinference_b200.priors import mlp, utils as su

T, B, G, F = 64, 256, 8, 18


def _hp(u):
    """The shipped BNN-prior configuration (reference tabular.py:47-70 / TabularEvalSimple.ipynb:154-176)."""
    return (lambda: 3, u.scaled_beta_sampler_f(2, 4, 150, 2), torch.nn.Tanh, u.gamma_sampler_f(3.62, .0677),
            u.gamma_sampler_f(1.87, .0528), lambda: 0.0, True, u.scaled_beta_sampler_f(1, 1.6, 18, 2), None, False, None,
            None, None, True, True, lambda n: ([], []), 0.0)


def _stats(x, y):
    x, y = x.double().cpu(), y.double().cpu()
    used = (x.abs().sum(0) > 0).sum(-1).double()
    xc, yc = x - x.mean(0), y - y.mean(0)
    corr = (xc * yc.unsqueeze(-1)).sum(0) / (xc.norm(dim=0) * yc.norm(dim=0).unsqueeze(-1) + 1e-12)
    halves_monotone = all(((y[k::2, i].diff() >= 0).all() or (y[k::2, i].diff() <= 0).all()) for i in range(y.shape[1]) for k in (0, 1))
    return dict(ymean=y.mean(0), used=used, maxcorr=corr.abs().max(-1).values, xscale=x.std(0).sum(-1) / used.clamp(min=1),
                halves_monotone=halves_monotone)


def _seed(s):
    np.random.seed(s); random.seed(s); torch.manual_seed(s)


def _reference_batch(seed):
    """_stats of the reference prior's batch drawn after _seed(seed)."""
    gold = os.path.join(os.path.dirname(__file__), "golden", "host_reference.pt")
    return torch.load(gold, weights_only=False)["mlp_prior"][seed]


def _check(ours, ref):
    # identical host stream => identical per-dataset feature counts and input scaling, exactly balanced median split
    assert torch.equal(ours["used"], ref["used"])
    assert torch.equal(ours["ymean"], ref["ymean"]) and float(ours["ymean"].mean()) == pytest.approx(0.5, abs=0.01)
    assert torch.allclose(ours["xscale"], ref["xscale"], rtol=1e-4)
    assert ours["halves_monotone"] and ref["halves_monotone"]          # order_by_y: both interleaved halves are sorted
    # function class: how predictable y is from the best single feature (two-sample z test on the mean, 4 sigma)
    a, b = ours["maxcorr"], ref["maxcorr"]
    se = (a.var() / len(a) + b.var() / len(b)).sqrt()
    assert abs(a.mean() - b.mean()) <= 4 * se, (float(a.mean()), float(b.mean()), float(se))
    assert abs(a.std() - b.std()) <= 0.05


def test_vectorised_mlp_prior_matches_reference_distribution_cpu():
    ref = _reference_batch(1)
    _seed(1)
    hp = _hp(su)
    x, y, _ = mlp._get_batch_vectorized(mlp._draw_model_specs(B // G, hp), G, T, F, 'cpu', hp, 'normal', 1)
    assert x.shape == (T, B, F) and y.shape == (T, B) and set(y.unique().tolist()) <= {0.0, 1.0}
    _check(_stats(x, y), ref)


def test_per_model_fallback_sees_the_same_models_after_replay():
    """When the vectorised path cannot be used (categorical features), the already-consumed host draws are replayed."""
    hp = _hp(su)
    _seed(3)
    specs = mlp._draw_model_specs(5, hp)
    rp = mlp._replay_hyperparameters(hp, specs)
    again = mlp._draw_model_specs(5, rp)
    assert [(s["hidden_dim"], s["num_features_used"], s["init_std"], s["noise_std"]) for s in specs] == \
           [(s["hidden_dim"], s["num_features_used"], s["init_std"], s["noise_std"]) for s in again]


@pytest.mark.gpu
def test_mlp_prior_device_path_matches_reference_distribution(cuda_device):
    ref = _reference_batch(2)
    _seed(2)
    x, y, t = mlp.get_batch(B, T, F, device='cuda:0', hyperparameters=_hp(su), batch_size_per_gp_sample=G)
    assert x.is_cuda and x.shape == (T, B, F) and torch.equal(y, t)
    _check(_stats(x, y), ref)
    # uniform causes and the regression variant (no binarisation) run through the same chain
    hp = list(_hp(su)); hp[6] = False
    x2, y2, _ = mlp.get_batch(32, 40, F, device='cuda:0', hyperparameters=tuple(hp), batch_size_per_gp_sample=4, sampling='uniform')
    assert torch.isfinite(x2).all() and torch.isfinite(y2).all() and y2.unique().numel() > 2
