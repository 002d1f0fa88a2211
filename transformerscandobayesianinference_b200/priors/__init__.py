"""Prior samplers of the PFN hot path (reference priors/): fast_gp, fast_gp_mix, mlp, stroke, omniglot, pyro (+ ridge as a tiny test prior).
Unlike the reference's `priors/__init__.py:1`, importing this package does not import gpytorch / botorch / pyro."""
from . import fast_gp, fast_gp_mix, mlp, omniglot, pyro, ridge, stroke, utils, prior  # noqa: F401
