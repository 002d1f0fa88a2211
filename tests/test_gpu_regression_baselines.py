"""Ridge baseline, exact GP (evaluate and sample) and binarized priors on the device: csrc/regression_baselines.cu against
the fp64 oracle element by element (oracle/regression_baselines_oracle.py bounds) and against the unmodified reference's
results (tests/golden/regression_baselines.pt), at the reference's __main__ shapes and at every edge the kernels branch
on."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import regression_baselines_oracle as O
from transformerscandobayesianinference_b200 import _lib as L
from transformerscandobayesianinference_b200 import train as train_mod
from transformerscandobayesianinference_b200.priors import binarized_regression as BR
from transformerscandobayesianinference_b200.priors import fast_gp, gp, ridge
from transformerscandobayesianinference_b200.priors.utils import _Deferred

GOLDEN = torch.load("tests/golden/regression_baselines.pt", weights_only=False)


def _ridge_device(x, y, target, alpha, dev):
    """x [B,T,F], y / target [B,T] -> pred, sq_err [B,T] fp64 numpy, NaN-prefilled outputs."""
    xb, yb, tb = (torch.as_tensor(v, dtype=torch.float32).to(dev).contiguous() for v in (x, y, target))
    pred = torch.full(yb.shape, float("nan"), dtype=torch.float64, device=dev)
    sq = torch.full_like(pred, float("nan"))
    L.ridge_prefix(xb, yb, tb, alpha, pred, sq)
    return pred.cpu().numpy(), sq.cpu().numpy()


def _check_ridge(x, y, target, alpha, dev, datasets=None):
    """Device against the oracle on every prefix of the given datasets; returns the device's sq_err."""
    x, y, target = (np.asarray(v, dtype=np.float32) for v in (x, y, target))      # what the kernel reads
    pred, sq = _ridge_device(x, y, target, alpha, dev)
    assert np.isnan(pred[:, 0]).all() and np.isnan(sq[:, 0]).all()
    for b in range(x.shape[0]) if datasets is None else datasets:
        p_ref, _, info = O.ridge_prefix_ref(x[b], y[b], target[b], alpha)
        gap = np.abs(pred[b, 1:] - p_ref[1:])
        bound = O.ridge_bound(info)[1:]
        assert np.all(gap <= bound), (b, int(np.argmax(gap / bound)) + 1, (gap / bound).max())
    return sq


@pytest.mark.parametrize("case", range(len(GOLDEN["ridge"])))
def test_ridge_matches_the_oracle_and_the_reference(case, cuda_device):
    c = GOLDEN["ridge"][case]
    x, y, yn = (c[k].transpose(0, 1).numpy() for k in ("x", "y", "y_non_noisy"))
    F = x.shape[2]
    sq = _check_ridge(x, y, yn, c["alpha"], cuda_device)
    t0 = 1 if c["alpha"] > 0 else F + 2                  # alpha = 0, rank deficient: sklearn's own rounding decides
    gap = np.abs(np.sqrt(sq[:, t0:]) - np.sqrt(c["elem"][t0:].T.numpy()))
    assert gap.max() <= 1e-9, gap.max()
    losses, _ = ridge.evaluate(c["x"], c["y"], c["y_non_noisy"], alpha=c["alpha"])
    assert losses.dtype == torch.float64 and losses.shape == (x.shape[1],) and losses[0] == 0
    np.testing.assert_allclose(losses[t0:].numpy(), c["losses"][t0:].numpy(), rtol=1e-8, atol=1e-14)


@pytest.mark.parametrize("alpha", [0.0, 1e-3])
@pytest.mark.parametrize("F", [1, 7, 64])
def test_ridge_edges_against_the_oracle(F, alpha, cuda_device):
    """t = 1, every t <= F (rank deficient), t = F + 1 and beyond, F at its limit, an odd F."""
    torch.manual_seed(F)
    T = F + 6
    x = torch.rand(3, T, F, dtype=torch.float64).numpy()
    y = (x @ torch.randn(F, dtype=torch.float64).numpy() * .1 + .01 * np.random.default_rng(F).normal(size=(3, T)))
    _check_ridge(x, y, y, alpha, cuda_device)


def test_ridge_at_the_reference_main_shape(cuda_device):
    torch.manual_seed(0)
    x, y, yn = ridge.get_batch(1000, 10, 10, noisy_std=.01)
    xb, yb, tb = (v.transpose(0, 1).numpy() for v in (x, y, yn))
    _check_ridge(xb, yb, tb, .01, cuda_device, datasets=range(0, 1000, 37))
    losses, secs = ridge.evaluate(x, y, yn, alpha=.01)
    sq = _ridge_device(xb, yb, tb, .01, cuda_device)[1]
    np.testing.assert_allclose(losses[1:].numpy(), sq[:, 1:].mean(0), rtol=1e-12)
    assert secs > 0


def _gp_device(x, y, ls, dev):
    xb = torch.as_tensor(x, dtype=torch.float32).to(dev).contiguous()
    yb = torch.as_tensor(y, dtype=torch.float32).to(dev).contiguous()
    mean = torch.full(yb.shape, float("nan"), dtype=torch.float64, device=dev)
    var, status = torch.full_like(mean, float("nan")), torch.full((xb.shape[0],), -1, dtype=torch.int32, device=dev)
    L.exact_gp_evaluate(xb, yb, ls, O.ALPHA_GP, mean, var, status)
    return mean.cpu().numpy(), var.cpu().numpy(), status.cpu().numpy()


def _check_gp(x, y, ls, dev):
    mean, var, status = _gp_device(x, y, ls, dev)
    assert (status == 0).all() and np.isnan(mean[:, 0]).all()
    for b in range(x.shape[0]):
        m, v, st, info = O.exact_gp_ref(x[b], y[b], ls)
        bm, bv = O.exact_gp_bound(info)
        assert st == 0
        assert np.all(np.abs(mean[b, 1:] - m[1:]) <= bm[1:]), b
        assert np.all(np.abs(var[b, 1:] - v[1:]) <= bv[1:]), b
    return mean, var


@pytest.mark.parametrize("case", range(len(GOLDEN["gp"])))
def test_gp_matches_the_oracle_and_the_reference(case, cuda_device):
    c = GOLDEN["gp"][case]
    x, y = c["x"].transpose(0, 1).numpy(), c["y"].transpose(0, 1).numpy()
    _check_gp(x, y, c["length_scale"], cuda_device)
    for use_mse, key in ((False, "nll"), (True, "mse")):
        losses, _ = gp.evaluate(c["x"], c["y"], c["y"], use_mse=use_mse, length_scale=c["length_scale"])
        bounds = []
        for b in range(x.shape[0]):
            m, v, _, info = O.exact_gp_ref(x[b], y[b], c["length_scale"])
            bounds.append(O.gp_loss_bound(m, v, y[b], *O.exact_gp_bound(info), use_mse))
        bound = np.mean(bounds, 0)[1:] * 2 + 1e-12                 # device's error plus the reference's
        assert losses[0] == 0 and np.all(np.abs(losses[1:].numpy() - c[key][1:].numpy()) <= bound), key


def test_gp_at_the_reference_main_shape_and_the_length_limit(cuda_device):
    torch.manual_seed(1)
    x, y, _ = gp.get_batch(1000, 10, 10, noisy_std=.6)
    assert x.shape == (10, 1000, 10) and y.shape == (10, 1000) and x.is_cuda and y.dtype == torch.float32
    losses, _ = gp.evaluate(x, y, y)
    assert losses.shape == (10,) and torch.isfinite(losses).all()
    _check_gp(x.transpose(0, 1)[:20].cpu().numpy(), y.transpose(0, 1)[:20].cpu().numpy(), .6, cuda_device)
    # T = 128 in 1-D at .6: a numerically singular kernel matrix, the variance-clamped regime
    x, y, _ = gp.get_batch(3, 128, 1)
    _check_gp(x.transpose(0, 1).cpu().numpy(), y.transpose(0, 1).cpu().numpy(), .6, cuda_device)
    assert torch.isfinite(gp.evaluate(x, y, y)[0]).all()
    with pytest.raises(ValueError, match="129 exceeds 128"):
        gp.evaluate(torch.rand(129, 2, 1), torch.rand(129, 2), torch.rand(129, 2))


def test_gp_raises_where_the_reference_raises(cuda_device):
    r = GOLDEN["gp_raise"]
    with pytest.raises(ValueError, match=f"dataset {r['dataset']}, t={r['t']}: a non-finite input"):
        gp.evaluate(r["x"], r["y"], r["y"])
    # the kernel's own status: the NaN row's pivot fails, so the fit of the prefix that contains it does
    _, _, status = _gp_device(r["x"].transpose(0, 1).numpy(), r["y"].transpose(0, 1).numpy(), .6, cuda_device)
    assert status.tolist() == [0, 0, 8, 0]
    y = r["y"].clone()
    y[4, 1] = float("inf")
    x = torch.rand_like(r["x"])
    with pytest.raises(ValueError, match="dataset 1, t=5: a non-finite input"):
        gp.evaluate(x, y, y)


def _sample(x, z, ls, dev):
    B, T, _ = x.shape
    out = torch.empty(B, T, device=dev)
    rank = torch.empty(B, dtype=torch.int32, device=dev)
    factor = torch.full((B, T, T), float("nan"), dtype=torch.float64, device=dev)
    perm = torch.empty(B, T, dtype=torch.int32, device=dev)
    L.exact_gp_sample(x, z, ls, out, rank, factor, perm)
    return out, rank, factor, perm


@pytest.mark.parametrize("F, ls, T", [(1, .6, 128), (1, .1, 128), (10, .6, 60), (3, .6, 1)])
def test_sampler_factor_and_draw(F, ls, T, cuda_device):
    torch.manual_seed(2)
    x, z = torch.rand(4, T, F, device=cuda_device), torch.randn(4, T, device=cuda_device)
    out, rank, factor, perm = _sample(x, z, ls, cuda_device)
    for b in range(4):
        xb = x[b].cpu().numpy()
        K = O.rbf_matrix(xb, xb, ls)
        Fb, pb, r = factor[b].cpu().numpy(), perm[b].cpu().numpy(), int(rank[b])
        assert sorted(pb.tolist()) == list(range(T)) and np.all(Fb[:, r:] == 0)
        assert np.all(np.triu(Fb[pb], 1) == 0)                      # P^T (P L) is lower triangular
        assert np.abs(Fb @ Fb.T - K).max() <= 4 * T * O.EPS        # stops at a remaining diagonal <= T eps
        y = Fb @ z[b].double().cpu().numpy()
        assert np.abs(out[b].cpu().numpy() - y).max() <= 2 ** -23 * (np.abs(y).max() + 1e-30)
        _, _, r_ref = O.pivoted_cholesky_ref(xb, ls)
        assert abs(r - r_ref) <= 2
    if (F, ls) == (1, .6):
        assert int(rank.max()) < 40                                 # singular K: the rank is the numerical one


def test_sampler_covariance_matches_the_kernel(cuda_device):
    torch.manual_seed(3)
    N, T = 40000, 8
    x = torch.rand(1, T, 2, device=cuda_device).expand(N, T, 2).contiguous()
    out, _, _, _ = _sample(x, torch.randn(N, T, device=cuda_device), .6, cuda_device)
    cov = (out.double().T @ out.double() / N).cpu().numpy()
    K = O.rbf_matrix(x[0].cpu().numpy(), x[0].cpu().numpy(), .6)
    assert np.abs(cov - K).max() <= 6 * math.sqrt(2.0 / N)
    y0 = gp.get_batch(2, T, 2, x=x[:2], z=torch.zeros(2, T))[1]
    assert torch.all(y0 == 0)


def test_binarized_labels(cuda_device):
    torch.manual_seed(5)
    x, labels, target = BR.regression_prior_to_binary(fast_gp.get_batch)(64, 20, 2, device=cuda_device)
    assert labels is target and set(labels.unique().tolist()) <= {0., 1.} and labels.shape == (20, 64)
    xs, zs, u = torch.rand(8, 20, 2, device=cuda_device), torch.randn(8, 20, device=cuda_device), torch.rand(20, 8,
                                                                                                           device=cuda_device)
    _, y, _ = fast_gp.get_batch(8, 20, 2, device=cuda_device, x=xs, z=zs)
    _, lab, _ = BR.regression_prior_to_binary(fast_gp.get_batch)(8, 20, 2, device=cuda_device, x=xs, z=zs, u=u,
                                                                 assert_on=True)
    assert torch.equal(lab, (u < torch.sigmoid(y)).float())


def test_binarized_labels_follow_an_escalated_y(cuda_device):
    """A deferred pivot check that fails re-samples y in place at hand-off; the labels must come from that final y."""
    torch.manual_seed(4)
    T = 48
    hps = {"noise": 0., "outputscale": 1., "lengthscale": .5}
    xs, zs, u = torch.rand(3, T, 1, device=cuda_device), torch.randn(3, T, device=cuda_device), torch.rand(T, 3,
                                                                                                         device=cuda_device)
    info = torch.empty(3, dtype=torch.int32, device=cuda_device)
    L.gp_sample(xs, zs, torch.full((3, 1), .5, device=cuda_device), torch.ones(3, device=cuda_device),
                torch.zeros(3, device=cuda_device), 0.0, L.KERNEL_RBF, torch.empty(3, T, device=cuda_device),
                torch.empty(3, T, T, device=cuda_device), info)
    assert bool(info.any())                                         # jitter 0 fails: the check must escalate
    y_final = fast_gp.get_batch(3, T, 1, device=cuda_device, hyperparameters=hps, x=xs, z=zs)[1]
    get = BR.regression_prior_to_binary(fast_gp.get_batch)
    _Deferred.active = True
    try:
        _, labels, _ = get(3, T, 1, device=cuda_device, hyperparameters=hps, x=xs, z=zs, u=u)
        checks = _Deferred.collect()
    finally:
        _Deferred.active = False
    assert len(checks) == 2
    torch.cuda.synchronize()
    assert set(labels.unique().tolist()) <= {0., 1.}                # valid before hand-off too
    for chk in checks:
        chk()
    assert torch.equal(labels, (u < torch.sigmoid(y_final)).float())


def test_binarized_fast_gp_trains_under_bce(cuda_device):
    torch.manual_seed(6)
    from transformerscandobayesianinference_b200 import encoders, utils
    total_loss, _, _ = train_mod.train(
        BR.Binarized_fast_gp_dataloader, train_mod.Losses.bce, encoders.Linear, emsize=64, nhid=128, nlayers=2, nhead=2,
        dropout=0.0, epochs=1, steps_per_epoch=2, batch_size=16, bptt=20, lr=1e-3, warmup_epochs=1,
        y_encoder_generator=encoders.Linear, extra_prior_kwargs_dict={"num_features": 1},
        single_eval_pos_gen=utils.get_weighted_single_eval_pos_sampler(15), verbose=False)
    assert math.isfinite(total_loss)
