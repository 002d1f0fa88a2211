"""Bayesian-NN prior on the device (csrc/bnn_prior.cu through pfn_bnn_prior and priors.pyro): every class decision and the
standardised inputs against the fp64 oracle through the kernel's own draws, the distribution of the draws, bitwise
independence of a dataset from its batch, training under Losses.bce, and the generic-callable path."""
import math

import numpy as np
import pytest
import scipy.stats as st
import torch

from oracle import bnn_oracle as O
from transformerscandobayesianinference_b200 import priors, train as T
from transformerscandobayesianinference_b200 import mcmc_svi_transformer_on_bayesian as M
from transformerscandobayesianinference_b200.priors import pyro as P

pytestmark = pytest.mark.gpu
SPECS = [(3, 5), (8, 64), (2, 7)]


@pytest.mark.parametrize("F,E", SPECS)
def test_decisions_and_standardisation_match_the_oracle(cuda_device, F, E):
    B, T = 64, 300
    x, y, w, xr, u = P.sample_bnn_prior(B, T, F, E, cuda_device, seed=123 + E, return_draws=True)
    assert x.shape == (T, B, F) and y.shape == (T, B) and w.shape == (B, O.dim(F, E)) and x.dtype == y.dtype == torch.float32
    p0, y_ref, x_ref = O.prior_forward_ref(w.cpu(), xr.cpu(), u.cpu(), F, E)
    # the kernel forms the probability in fp64 from the same fp32 draws: a decision may differ only where u lies within
    # the rounding of p0 (1e-12 covers the ~2 E F ulp of the two dot products and the exp)
    near = (u.cpu() - p0).abs() <= 1e-12
    assert (y.cpu().double() == y_ref)[~near].all() and near.sum() <= 1
    assert set(y.unique().tolist()) <= {0.0, 1.0}
    # standardised x: fp64 statistics, one rounding to fp32 (2^-24 relative) plus the statistics' own rounding
    err = (x.cpu().double() - x_ref).abs()
    bound = 2.0 ** -24 * x_ref.abs() + 1e-12
    assert (err <= bound).all(), float((err - bound).max())


def test_draws_are_standard_normal_and_classes_balanced(cuda_device):
    F, E, B, T = 3, 5, 512, 300
    x, y, w, xr, u = P.sample_bnn_prior(B, T, F, E, cuda_device, seed=7, return_draws=True)
    for name, v in (("weights", w), ("x_raw", xr)):
        v = v.double().cpu().numpy().ravel()
        se = 1 / math.sqrt(len(v))
        assert abs(v.mean()) <= 5 * se and abs(v.var() - 1) <= 5 * math.sqrt(2) * se, (name, v.mean(), v.var())
        assert abs((v ** 4).mean() - 3) <= 5 * math.sqrt(96) * se
        assert st.kstest(v[:200000], "norm").pvalue > 1e-4, name
    uu = u.cpu().numpy().ravel()
    assert st.kstest(uu, "uniform").pvalue > 1e-4 and uu.min() >= 0 and uu.max() < 1
    # distinct datasets have distinct weights and inputs
    assert len({float(v) for v in w[:, 0]}) >= B - 2 and len({float(v) for v in xr[0, :, 0]}) >= B - 2
    # by the sign symmetry of the weights each class has probability 1/2; datasets are independent
    per_dataset = y.mean(0).double().cpu().numpy()
    assert abs(per_dataset.mean() - 0.5) <= 5 * per_dataset.std(ddof=1) / math.sqrt(B)
    assert per_dataset.std() > 0.05                              # and a dataset's own balance varies with its weights


def test_a_dataset_does_not_depend_on_its_batch(cuda_device):
    F, E, T = 3, 5, 100
    x, y = P.sample_bnn_prior(16, T, F, E, cuda_device, seed=99)
    for b in (0, 5, 15):
        x1, y1 = P.sample_bnn_prior(1, T, F, E, cuda_device, seed=99, dataset_offset=b)
        assert torch.equal(x1[:, 0], x[:, b]) and torch.equal(y1[:, 0], y[:, b])
    x2, _ = P.sample_bnn_prior(16, T, F, E, cuda_device, seed=100)
    assert not torch.equal(x2, x)


def test_get_batch_and_model_draws(cuda_device):
    spec = M.get_default_model_spec('small')
    torch.manual_seed(0)
    x, y, t = P.get_batch(32, 50, batch_size_per_gp_sample=8, model=lambda: M.BayesianModel(spec), device=cuda_device)
    assert x.shape == (50, 32, 3) and y.shape == (50, 32) and t is y and x.is_cuda
    torch.manual_seed(0)
    x2, _, _ = P.get_batch(32, 50, batch_size_per_gp_sample=8, model=lambda: M.BayesianModel(spec), device=cuda_device)
    assert torch.equal(x, x2)                                    # reproducible under torch.manual_seed
    with pytest.raises(AssertionError, match="divisible"):
        P.get_batch(32, 50, batch_size_per_gp_sample=5, model=lambda: M.BayesianModel(spec), device=cuda_device)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        P.get_batch(32, 50, model=lambda: M.BayesianModel(spec), device='cpu')
    with pytest.raises(ValueError, match="above the limit"):
        P.sample_bnn_prior(2, 10, 8, 200, cuda_device)
    xs, obs = M.BayesianModel(spec, device='cuda')(seq_len=40)
    assert xs.shape == (40, 3) and obs.shape == (40,)
    X, Y = M.generate_toy_data(M.BayesianModel(spec, device='cuda'), 30)
    assert X.shape == (100, 30, 3) and Y.shape == (100, 30) and X.device.type == 'cpu'
    assert len({float(v) for v in X[:, 0, 0]}) == 100


def test_generic_callable_returns_the_reference_shapes(cuda_device):
    class Toy:
        def __call__(self, seq_len=1):
            x = torch.randn(seq_len, 4)
            return x, (x[:, 0] > 0).float()

    x, y, t = P.get_batch(8, 20, batch_size_per_gp_sample=2, model=Toy, device=cuda_device)
    assert x.shape == (20, 8, 4) and y.shape == (20, 8) and x.is_cuda and t is y
    assert x.mean(0).abs().max() < 1e-5


def test_dataloader_trains_under_bce(cuda_device):
    torch.manual_seed(1)
    spec = M.get_default_model_spec('small')
    tr = T.build_trainer(priors.pyro.DataLoader, T.Losses.bce, T.encoders.Linear, emsize=64, nhid=128, nlayers=2, nhead=2,
                         dropout=0.0, epochs=4, steps_per_epoch=8, batch_size=32, bptt=40, lr=1e-3, warmup_epochs=1,
                         y_encoder_generator=T.encoders.Linear, gpu_device=str(cuda_device),
                         single_eval_pos_gen=M.get_weighted_single_eval_pos_sampler(30),
                         extra_prior_kwargs_dict={'num_outputs': 1, 'num_features': 3, 'fuse_x_y': False,
                                                  'model': lambda: M.BayesianModel(spec)})
    losses = []
    for _ in range(4):
        losses.append(tr.train_epoch()[0])
        tr.scheduler.step()
    print("epoch losses", losses)
    assert all(math.isfinite(l) for l in losses) and losses[-1] <= losses[0] + 0.02
