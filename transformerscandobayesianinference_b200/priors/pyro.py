"""`priors.pyro` (reference priors/pyro.py): datasets drawn from a Bayesian model given as a zero-argument callable.

The reference calls `config['model']()` once per group of datasets and the returned pyro module once per dataset in a
Python loop.  When the callable returns this package's `BayesianModel` (mcmc_svi_transformer_on_bayesian.py: a
two-layer network with N(0, 1) weights and inputs and a categorical observation) the whole batch comes from one launch of
csrc/bnn_prior.cu instead: weights, inputs, logits, class draw and the standardisation of x per dataset and feature.  As
pyro re-draws the weights on every call of the model, every dataset has its own weights; `batch_size_per_gp_sample` only
sets how many model objects are constructed.  The random numbers are counter-based hashes of one seed per batch drawn
from torch's CPU generator, so a batch is reproducible under `torch.manual_seed` and costs no device sync; the
distribution is the reference's, the individual draws are not (torch's stream is not replayed).

Any other callable is run as the reference runs it, one call per dataset, and the results are stacked (host glue for
custom modules, not a sampler).
"""
import torch

from .. import _lib as L
from ..utils import default_device
from .utils import get_batch_to_dataloader, normalize_data


def sample_bnn_prior(batch_size, seq_len, num_features, embed, device, seed=None, dataset_offset=0, return_draws=False):
    """x [seq_len, B, F] fp32 (standardised), y [seq_len, B] fp32 from one kernel launch.  With return_draws also the
    oracle hook (weights [B, d] fp32, x_raw [seq_len, B, F] fp32, u [seq_len, B] fp64)."""
    d = embed * num_features + 3 * embed + 2
    if d > L.BNN_MAX_D:
        raise ValueError(f"priors.pyro: the network has d = E F + 3 E + 2 = {d} weights, above the limit of {L.BNN_MAX_D}")
    dev = L.cuda_device(device, "priors.pyro draws BayesianModel datasets with the sm_90a kernel of csrc/bnn_prior.cu")
    seed = L.draw_seed(seed)
    with L.on_device(dev):
        x = torch.empty(seq_len, batch_size, num_features, dtype=torch.float32, device=dev)
        y = torch.empty(seq_len, batch_size, dtype=torch.float32, device=dev)
        draws = (None, None, None)
        if return_draws:
            draws = (torch.empty(batch_size, d, dtype=torch.float32, device=dev), torch.empty_like(x),
                     torch.empty(seq_len, batch_size, dtype=torch.float64, device=dev))
        L.bnn_prior(x, y, seed, embed, dataset_offset, *draws)
    return (x, y) + (draws if return_draws else ())


@torch.no_grad()
def get_batch(batch_size, seq_len, batch_size_per_gp_sample=None, device=default_device, **config):
    """-> x [seq_len, B, F], y [seq_len, B], y (reference :10-34).  `config['model']` is a zero-argument callable; it is
    called batch_size / batch_size_per_gp_sample times (default group size: batch_size // 16)."""
    from ..mcmc_svi_transformer_on_bayesian import BayesianModel
    group = batch_size_per_gp_sample or batch_size // 16
    assert batch_size % group == 0, 'Please choose a batch_size divisible by batch_size_per_gp_sample.'
    models = [config['model']() for _ in range(batch_size // group)]
    shapes = {(m.num_features, m.embed) if isinstance(m, BayesianModel) else None for m in models}
    if len(shapes) == 1 and None not in shapes:
        (num_features, embed), = shapes
        x, y = sample_bnn_prior(batch_size, seq_len, num_features, embed, device)
        return x, y, y

    # any other model: one call per dataset, `group` datasets per model object, then x standardised over the sequence axis
    draws = [model(seq_len=seq_len) for model in models for _ in range(group)]
    x = torch.stack([d[0] for d in draws], 1).detach().to(device)
    y = torch.stack([d[1] for d in draws], 1).squeeze(-1).detach().to(device)
    return normalize_data(x), y, y


DataLoader = get_batch_to_dataloader(get_batch)
DataLoader.num_outputs = 1
