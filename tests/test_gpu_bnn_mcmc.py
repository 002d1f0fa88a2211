"""NUTS baseline of the Bayesian NN on the device (csrc/bnn_mcmc.cu through pfn_bnn_mcmc): the potential and its gradient
against the fp64 oracle, trajectory parity with the CPU NUTS restatement with the state in shared memory and in the global
workspace, the posterior predictive against importance sampling, bitwise reproducibility, and `eval_mcmc`'s conventions."""
import math

import numpy as np
import pytest
import torch

from oracle import bnn_oracle as O
from oracle.gp_mcmc_oracle import nuts_chain
from transformerscandobayesianinference_b200 import _lib as L
from transformerscandobayesianinference_b200 import mcmc_svi_transformer_on_bayesian as M
from transformerscandobayesianinference_b200.priors import pyro as P

pytestmark = pytest.mark.gpu
DIAG = {n: i for i, n in enumerate(L.GP_MCMC_DIAG_NAMES)}
SMALL, BIG, ODD = (3, 5), (8, 64), (5, 53)            # d = 32 (shared memory), 706 and 426 (global workspace)


def _spec(FE):
    return {'num_features': FE[0], 'embed': FE[1]}


def _toy(FE, N, T, device, seed):
    """N datasets of T rows from the prior, as eval_mcmc sees them: X [N, T, F], y [N, T]."""
    x, y = P.sample_bnn_prior(N, T, FE[0], FE[1], device, seed=seed)
    return x.transpose(0, 1).contiguous(), y.transpose(0, 1).contiguous()


def _uses_workspace(FE, n):
    return L.bnn_mcmc_workspace(L.bnn_mcmc_desc(1, n, 0, FE[0], FE[1], 1, 1, 0)) > 0


@pytest.mark.parametrize("n", [1, 2, 100])
@pytest.mark.parametrize("FE", [SMALL, BIG, ODD])
def test_potential_and_gradient_match_the_oracle(cuda_device, FE, n):
    F, E = FE
    N, m, d = 3, 7, O.dim(F, E)
    X, y = _toy(FE, N, n + m, cuda_device, seed=n + d)
    g = torch.Generator().manual_seed(d + n)
    th0 = torch.randn(N, d, generator=g, dtype=torch.float64) * torch.tensor([0.3, 1.0, 2.0], dtype=torch.float64)[:, None]
    assert _uses_workspace(FE, n) == (FE != SMALL)
    r = M.sample_bnn_posterior(X[:, :n], y[:, :n], X[:, n:], _spec(FE), 0, 0, seed=0, init=th0)
    r = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in r.items()}
    assert (r["diag"][:, DIAG["evals"]] == 1).all() and (r["diag"][:, DIAG["not_pd"]] == 0).all()
    assert torch.equal(r["samples"][:, 0], th0) and (r["step_size"] == 0).all()
    Xd, yd = X.double().cpu(), y.cpu()
    for b in range(N):
        U, gr = O.potential_value_and_grad_ref(Xd[b, :n], yd[b, :n], th0[b].numpy(), F, E)
        assert abs(r["potential"][b].item() - U) <= 1e-10 * (1 + abs(U)), (b, r["potential"][b].item(), U)
        assert np.abs(r["grad"][b].numpy() - gr).max() <= 1e-8 * (1 + np.linalg.norm(gr)), b
        p1 = O.predictive_ref(th0[b], Xd[b, n:], F, E)
        assert (r["probs"][b, 0] - p1).abs().max().item() <= 1e-12


@pytest.mark.parametrize("FE,n,depth,chains,from_init", [
    pytest.param(SMALL, 10, 10, 6, False, id="FE0-10-10-6"), pytest.param(SMALL, 10, 2, 6, False, id="FE1-10-2-6"),
    pytest.param(BIG, 20, 4, 4, False, id="FE2-20-4-4"), pytest.param(BIG, 20, 2, 4, False, id="FE3-20-2-4"),
    pytest.param(SMALL, 10, 2, 6, True, id="small-10-2-6-init")])
def test_trajectories_follow_the_cpu_restatement(cuda_device, FE, n, depth, chains, from_init):
    """40 iterations (warmup 30 with windows ending at 3, 26, 29, so one mass-matrix update and three step-size searches,
    then 10 samples) against oracle nuts_chain on the numpy potential: theta to 1e-6, the step size to 1e-6 relative and
    every tree depth.  The two differ in the order of their sums (the device adds per-thread partials), i.e. in the last
    bits of every energy, and a NUTS trajectory amplifies that: with trees of depth 4 and more (`small` at the full cap,
    about 20 leapfrog steps per iteration; `big`, d = 706 in the global workspace, capped at depth 4) the difference
    grows by roughly a factor of three per iteration, is about 1e-9 after 10 iterations and passes the tolerance after 16
    to 32, after which the two are different valid chains.  Every chain must agree through the first step-size search
    and 10 iterations; with the trees capped at depth 2 the amplification is small and at least half of the chains must
    agree through all 40 iterations, mass-matrix update included, with the state in shared memory (`small`) and in the
    global workspace (`big`).  A chain started from a caller's init draws its first momenta at the same keys as one that
    draws its initial point (the initial point takes no draws then)."""
    F, E = FE
    W, S, seed, d = 30, 10, 4321, O.dim(*FE)
    X, y = _toy(FE, chains, n, cuda_device, seed=17)
    assert _uses_workspace(FE, n) == (FE != SMALL)
    th0 = torch.randn(chains, d, generator=torch.Generator().manual_seed(9), dtype=torch.float64) if from_init else None
    r = M.sample_bnn_posterior(X, y, None, _spec(FE), S, W, seed=seed, max_tree_depth=depth, init=th0, trace=True)
    tr = r["trace"].cpu().numpy()
    Xd, yd = X.double().cpu().numpy(), y.cpu().numpy()
    agree, parted, at10 = 0, [], []
    for b in range(chains):
        if from_init:
            c = nuts_chain(O.potential_and_grad_np(Xd[b], yd[b], F, E), d, S, W, seed, b=b, t=n, init=th0[b].tolist(),
                           max_tree_depth=depth)
        else:
            c = O.bnn_chain_job((Xd[b], yd[b], F, E, S, W, seed, b, depth))
        dth = np.abs(c["trace"][:, :d] - tr[b, :, :d]).max(1)
        at10.append(float(dth[10]))
        bad = np.nonzero((dth > 1e-6) | (c["trace"][:, d + 1] != tr[b, :, d + 1]) |
                         (np.abs(c["trace"][:, d] - tr[b, :, d]) > 1e-6 * c["trace"][:, d]))[0]
        if len(bad) == 0:
            agree += 1
            assert c["diag"]["leapfrog"] == r["diag"][b, DIAG["leapfrog"]].item()
        else:
            parted.append((b, int(bad[0]), float(dth[bad[0]])))
    print(f"{FE} depth cap {depth}: {agree} of {chains} chains agree in all {W + S} iterations, mean depth "
          f"{tr[:, :, d + 1].mean():.2f}, max |dtheta| at iteration 10 {max(at10):.1e}; "
          f"parted (chain, iteration, |dtheta|): {parted}")
    assert all(it >= 10 for _, it, _ in parted), parted
    if depth <= 2:
        assert agree >= chains / 2, parted


@pytest.mark.parametrize("FE,n", [((1, 1), 2), ((1, 1), 10), ((2, 2), 5)])
def test_posterior_predictive_matches_importance_sampling(cuda_device, FE, n):
    F, E = FE
    R, m, W, S = 256, 4, 200, 200
    X, y = _toy(FE, 1, n + m, cuda_device, seed=5 + n)
    ref = O.importance_predictive(X[0, :n].cpu(), y[0, :n].cpu(), X[0, n:].cpu(), F, E, num_draws=1 << 22, seed=1,
                                  device=cuda_device)
    assert ref["ess"] > 2e4, ref
    Xr, yr = X.repeat(R, 1, 1), y.repeat(R, 1)                # the same dataset in every slot: R chains with their own keys
    r = M.sample_bnn_posterior(Xr[:, :n], yr[:, :n], Xr[:, n:], _spec(FE), S, W, seed=77)
    assert r["diag"][:, DIAG["div_sampling"]].sum().item() <= 0.01 * R * S
    est = r["probs"].mean(1).cpu().numpy()                   # [R, m]: every chain's estimate
    se = np.sqrt(est.var(0, ddof=1) / R + ref["se"] ** 2)
    z = np.abs(est.mean(0) - ref["p1"]) / se
    print(f"{FE} n={n}: chains {est.mean(0)} importance sampling {ref['p1']} (ess {ref['ess']:.0f}) se {se} z {z}, "
          f"mean accept {r['accept'].mean().item():.3f}, depth-cap hits {r['diag'][:, DIAG['max_depth_hits']].sum().item()}")
    assert (z <= 5).all(), (est.mean(0), ref["p1"], se)
    # the drawn classes are Bernoulli draws of those probabilities
    obs = r["obs"].double().mean((0, 1)).cpu().numpy()
    assert (np.abs(obs - est.mean(0)) <= 5 * 0.5 / math.sqrt(R * S)).all()


@pytest.mark.parametrize("FE,depth", [(SMALL, 10), (ODD, 5)])
def test_a_chain_does_not_depend_on_its_launch(cuda_device, FE, depth):
    n, m, S, W = 12, 5, 15, 25
    X, y = _toy(FE, 9, n + m, cuda_device, seed=3)
    many = M.sample_bnn_posterior(X[:, :n], y[:, :n], X[:, n:], _spec(FE), S, W, seed=11, max_tree_depth=depth, trace=True)
    alone = M.sample_bnn_posterior(X[:1, :n], y[:1, :n], X[:1, n:], _spec(FE), S, W, seed=11, max_tree_depth=depth, trace=True)
    for k in ("samples", "probs", "obs", "potential", "grad", "step_size", "accept", "diag", "trace"):
        assert torch.equal(alone[k][0], many[k][0]), k
    again = M.sample_bnn_posterior(X[:, :n], y[:, :n], X[:, n:], _spec(FE), S, W, seed=11, max_tree_depth=depth)
    other = M.sample_bnn_posterior(X[:, :n], y[:, :n], X[:, n:], _spec(FE), S, W, seed=12, max_tree_depth=depth)
    assert torch.equal(again["samples"], many["samples"]) and torch.equal(again["diag"], many["diag"])
    assert not torch.equal(other["samples"], many["samples"])
    assert torch.isfinite(many["samples"]).all() and (many["diag"][:, DIAG["leapfrog"]] > 0).all()


@pytest.mark.parametrize("FE", [SMALL, ODD])
def test_outputs_do_not_depend_on_what_the_buffers_held(cuda_device, FE):
    F, E = FE
    N, n, m, S, W, d = 4, 8, 3, 10, 20, O.dim(*FE)
    X, y = _toy(FE, N, n + m, cuda_device, seed=8)
    xtr, ytr, xte = X[:, :n].contiguous(), y[:, :n].contiguous(), X[:, n:].contiguous()

    def launch(fill):
        f64 = dict(dtype=torch.float64, device=cuda_device)
        desc = L.bnn_mcmc_desc(N, n, m, F, E, S, W, 5, 5)
        per_chain = L.bnn_mcmc_workspace(desc)
        out = {"samples": torch.full((N, S, d), fill, **f64), "probs": torch.full((N, S, m), fill, **f64),
               "obs": torch.full((N, S, m), fill, dtype=torch.float32, device=cuda_device),
               "potential": torch.full((N,), fill, **f64), "grad": torch.full((N, d), fill, **f64),
               "trace": torch.full((N, W + S, d + 2), fill, **f64)}
        step, acc = torch.full((N,), fill, **f64), torch.full((N,), fill, **f64)
        diag = torch.full((N, 6), -7, dtype=torch.int32, device=cuda_device)
        ws = torch.full((N, per_chain), fill, **f64) if per_chain else None
        L.bnn_mcmc(xtr, ytr, xte, desc, out["samples"], step, acc, diag, workspace=ws, **{k: v for k, v in out.items() if k != "samples"})
        return dict(out, step_size=step, accept=acc, diag=diag)

    a, b = launch(float("nan")), launch(0.0)
    for k in a:
        assert torch.equal(a[k], b[k]) and not torch.isnan(a[k].double()).any(), k


@pytest.mark.parametrize("FE", [SMALL, ODD])
def test_warmup_only_returns_the_last_state(cuda_device, FE):
    """num_samples = 0 with warmup: the single output row is the state after the last warmup iteration, whatever the
    output buffers held, and the probabilities are formed at it."""
    N, n, m, W, d = 3, 8, 4, 12, O.dim(*FE)
    X, y = _toy(FE, N, n + m, cuda_device, seed=21)
    r = M.sample_bnn_posterior(X[:, :n], y[:, :n], X[:, n:], _spec(FE), 0, W, seed=6, max_tree_depth=4, trace=True)
    assert r["samples"].shape == (N, 1, d) and r["trace"].shape == (N, W, d + 2)
    assert torch.equal(r["samples"][:, 0], r["trace"][:, -1, :d]) and torch.isnan(r["accept"]).all()
    for b in range(N):
        p1 = O.predictive_ref(r["samples"][b, 0].cpu(), X[b, n:].double().cpu(), *FE)
        assert (r["probs"][b, 0].cpu() - p1).abs().max().item() <= 1e-12
    again = M.sample_bnn_posterior(X[:, :n], y[:, :n], X[:, n:], _spec(FE), 0, W, seed=6, max_tree_depth=4)
    assert torch.equal(again["samples"], r["samples"]) and torch.equal(again["obs"], r["obs"])


def test_eval_mcmc_follows_the_reference_conventions(cuda_device, tmp_path):
    spec = M.get_default_model_spec('small')
    X, y = M.generate_toy_data(M.BayesianModel(spec, device='cuda'), 40)
    X, y = X[:12], y[:12]
    sampler = lambda: M.BayesianModel(spec, device='cuda')
    nll, acc = M.eval_mcmc(X, y, 'cuda:0', sampler, 10, warmup_steps=30, num_pred_samples=20, seed=9)
    assert isinstance(nll, np.ndarray) and nll.shape == (12,) and acc.shape == (12,)
    assert np.isfinite(nll).all() and ((acc >= 0) & (acc <= 1)).all()
    r = M.sample_bnn_posterior(X[:, :10].cuda(), y[:, :10].cuda(), X[:, 10:].cuda(), spec, 20, 30, seed=9)
    assert r["obs"].shape == (12, 20, 30) and set(r["obs"].unique().tolist()) <= {0.0, 1.0}
    for b in (0, 7):
        means = r["obs"][b].mean(0).cpu()
        assert abs(nll[b] - torch.nn.BCELoss()(means, y[b, 10:]).item()) < 1e-6
        assert abs(acc[b] - (r["obs"][b].cpu() == y[b, 10:]).float().mean().item()) < 1e-6
    nll2, _ = M.eval_mcmc(X, y, 'cpu', sampler, 10, warmup_steps=30, num_pred_samples=20, seed=9)
    assert np.array_equal(nll, nll2)
    # the drivers write the reference's files
    M.training_samples('mcmc', X, y, sampler, [2, 7], steps=16, path_interfix=str(tmp_path))
    files, times, samples, means, conf = M.load_results(f'{tmp_path}/results_mcmc_16_training_samples', task='samples')
    assert list(samples) == [2, 7] and means.shape == (2,) and np.isfinite(means).all()
    # the transformer on the same data: all datasets in one forward pass
    _, _, model = M.get_model(sampler, dict(M.get_transformer_config(spec), epochs=4, steps_per_epoch=2, batch_size=16,
                                            emsize=64, nlayers=2, nhead=2, seq_len=120), device='cuda:0')
    tacc, tnll, elapsed = M.eval_transformer(X, y, 'cuda:0', model, 10)
    assert tacc.shape == (12,) and tnll.shape == (12,) and torch.isfinite(tnll).all() and elapsed > 0


def test_sizes_beyond_the_caps_raise(cuda_device):
    X, y = _toy(SMALL, 2, 20, cuda_device, seed=1)
    with pytest.raises(ValueError, match="above the sampler's limit"):
        M.sample_bnn_posterior(torch.zeros(2, 10, 8, device=cuda_device), y[:, :10], None, {'num_features': 8, 'embed': 200}, 5, 5, seed=0)
    with pytest.raises(ValueError, match="outside"):
        M.sample_bnn_posterior(torch.zeros(2, 2000, 3, device=cuda_device), torch.zeros(2, 2000, device=cuda_device), None,
                               _spec(SMALL), 5, 5, seed=0)
    with pytest.raises(ValueError, match="max_tree_depth"):
        M.sample_bnn_posterior(X, y, None, _spec(SMALL), 5, 5, seed=0, max_tree_depth=11)
    with pytest.raises(ValueError, match="features"):
        M.sample_bnn_posterior(X, y, None, _spec(BIG), 5, 5, seed=0)
