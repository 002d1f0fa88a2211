"""`priors.binarized_regression` (reference priors/binarized_regression.py): GP-classification priors, the draws of a
regression prior pushed through a sigmoid and a Bernoulli draw, for training binary classifiers under Losses.bce.

The labels are u < sigmoid(y) with u ~ U[0,1) drawn on y's device: the reference's `y.sigmoid().bernoulli()` in
distribution, not in torch's CPU random stream.  While a prefetching loader defers fast_gp's pivot check, a failed check
re-samples y in place when the batch is handed over; the labels are therefore formed at once and again after the deferred
checks of their batch (no host sync), so that the labels a consumer receives follow the final y.  A tensor derived from
the labels before hand-off (e.g. the loader's fused x/y input) is not updated."""
import torch

from . import fast_gp, fast_gp_mix
from .utils import again_after_deferred_checks, get_batch_to_dataloader


def regression_prior_to_binary(get_batch_function):

    def binarized_get_batch_function(*args, assert_on=False, u=None, **kwargs):
        """`u` (extension): uniforms of y's shape to draw the labels with, instead of drawing them on the device."""
        x, y, target_y = get_batch_function(*args, **kwargs)
        if assert_on:
            assert y is target_y, "y == target_y is assumed by this function"
        u = torch.rand_like(y) if u is None else u.to(y.device, y.dtype)
        labels = torch.empty_like(y)

        def label():
            if labels.is_cuda:
                for t in (y, u):
                    t.record_stream(torch.cuda.current_stream(labels.device))
            labels.copy_(u < torch.sigmoid(y))

        again_after_deferred_checks(label)
        return x, labels, labels

    return binarized_get_batch_function


Binarized_fast_gp_dataloader = get_batch_to_dataloader(regression_prior_to_binary(fast_gp.get_batch))
Binarized_fast_gp_dataloader.num_outputs = 1


Binarized_fast_gp_mix_dataloader = get_batch_to_dataloader(regression_prior_to_binary(fast_gp_mix.get_batch))
Binarized_fast_gp_mix_dataloader.num_outputs = 1
