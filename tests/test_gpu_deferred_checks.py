"""The deferred sampler checks cost no host sync: while the prefetching loader defers (`_Deferred.active`), the GP pivot
flags and the stroke rejection flag travel to pinned host memory and are read only when the collected checks run."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L
from transformerscandobayesianinference_b200.priors import fast_gp, stroke
from transformerscandobayesianinference_b200.priors.utils import _Deferred


def _draws(dev, gp):
    hps = {"noise": 1e-4, "outputscale": 1., "lengthscale": .6}
    return [fast_gp.get_batch(8, 100, 2, device=dev, hyperparameters=hps),
            stroke.get_batch(8, 11, num_features=100, num_outputs=2, device=dev),
            fast_gp.sample_gp(*gp)]


def test_deferred_checks_do_not_sync(cuda_device):
    dev = cuda_device
    torch.manual_seed(4)
    T = 48
    # dataset 1 has zero noise: a smooth RBF matrix on 48 points is numerically singular in fp32 => needs jitter
    gp = (torch.rand(3, T, 1, device=dev), torch.randn(3, T, device=dev), torch.full((3, 1), .5, device=dev),
          torch.ones(3, device=dev), torch.tensor([1e-2, 0., 1e-2], device=dev))
    info = torch.empty(3, dtype=torch.int32, device=dev)
    L.gp_sample(*gp, 0.0, L.KERNEL_RBF, torch.empty(3, T, device=dev), torch.empty(3, T, T, device=dev), info)
    assert bool(info.any())                        # so the sample_gp call below has to escalate its jitter
    y_sync = fast_gp.sample_gp(*gp)

    _Deferred.active = True
    try:
        _draws(dev, gp)                            # first calls outside the check: library load, pinned host blocks
        for check in _Deferred.collect():
            check()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = _draws(dev, gp)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        checks = _Deferred.collect()
    finally:
        _Deferred.active = False
    assert len(checks) == 3
    for check in checks:
        check()
    torch.cuda.synchronize()
    assert torch.isfinite(out[2]).all() and torch.allclose(out[2], y_sync, rtol=1e-5, atol=1e-6)
