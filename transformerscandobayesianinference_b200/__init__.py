"""transformerscandobayesianinference_b200 — a H100-native (sm_90a) engine for the PFN training hot path of
automl/TransformersCanDoBayesianInference, behind the reference's own Python module API.

    from transformerscandobayesianinference_b200 import train, transformer, bar_distribution, priors, encoders, utils

or, for unmodified notebooks that do `from train import train; import priors, encoders, ...`:

    import transformerscandobayesianinference_b200 as pfn; pfn.install_dropin()
"""
import importlib
import sys

__version__ = "0.1.0"

_DROPIN_MODULES = ("utils", "encoders", "positional_encodings", "bar_distribution", "transformer", "priors", "train")


def install_dropin():
    """Register this package's modules under the reference's top-level module names (train, transformer,
    bar_distribution, priors, encoders, positional_encodings, utils) so reference notebooks import them unchanged."""
    for name in _DROPIN_MODULES:
        mod = importlib.import_module(f"{__name__}.{name}")
        sys.modules[name] = mod
    sys.modules["priors.fast_gp"] = importlib.import_module(f"{__name__}.priors.fast_gp")
    sys.modules["priors.fast_gp_mix"] = importlib.import_module(f"{__name__}.priors.fast_gp_mix")
    sys.modules["priors.mlp"] = importlib.import_module(f"{__name__}.priors.mlp")
    sys.modules["priors.stroke"] = importlib.import_module(f"{__name__}.priors.stroke")
    sys.modules["priors.omniglot"] = importlib.import_module(f"{__name__}.priors.omniglot")
    sys.modules["priors.utils"] = importlib.import_module(f"{__name__}.priors.utils")
    sys.modules["priors.pyro"] = importlib.import_module(f"{__name__}.priors.pyro")
    sys.modules["mcmc_svi_transformer_on_bayesian"] = importlib.import_module(f"{__name__}.mcmc_svi_transformer_on_bayesian")
    return {name: sys.modules[name] for name in _DROPIN_MODULES}
