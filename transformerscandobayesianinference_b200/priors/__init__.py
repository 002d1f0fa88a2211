"""Prior samplers of the PFN hot path (reference priors/): fast_gp, gp, ridge, stroke, fast_gp_mix, mlp, omniglot,
binarized_regression and pyro, the modules of the reference's `priors/__init__.py:1`.  Unlike the reference, importing
this package imports none of gpytorch / botorch / pyro / sklearn."""
from . import binarized_regression, fast_gp, fast_gp_mix, gp, mlp, omniglot, pyro, ridge, stroke, utils, prior  # noqa: F401
