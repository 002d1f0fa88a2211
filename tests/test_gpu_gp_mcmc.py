"""Fully Bayesian GP baseline on the device (csrc/gp_mcmc.cu through pfn_gp_mcmc): the potential and its gradient against
the fp64 oracle, trajectory parity with the CPU NUTS restatement, the posterior against quadrature, bitwise
reproducibility, and the reference's `evaluate_` conventions."""
import math

import numpy as np
import pytest
import torch

from oracle import gp_mcmc_oracle as M
from oracle.gp_fit_oracle import gp_matern_ref
from transformerscandobayesianinference_b200 import _lib as L
from transformerscandobayesianinference_b200.priors import fast_gp_mix

pytestmark = pytest.mark.gpu
DIAG = {n: i for i, n in enumerate(L.GP_MCMC_DIAG_NAMES)}


@pytest.mark.parametrize("nu", [0.5, 1.5, 2.5])
@pytest.mark.parametrize("F", [1, 3, 5])
def test_potential_and_gradient_match_the_oracle(cuda_device, nu, F):
    g = torch.Generator().manual_seed(int(10 * nu) + 100 * F)
    B, T, ts = 4, 128, [1, 2, 17, 64, 100, 128]
    x = torch.rand(B, T, F, generator=g)
    x[0, 5], x[0, 40], x[0, 99] = x[0, 3], x[0, 10], x[0, 10]          # duplicate rows (r = 0 pairs)
    x[1, 1] = x[1, 0]
    y = torch.randn(B, T, generator=g)
    u0 = torch.cat([torch.randn(len(ts), B, F + 1, generator=g, dtype=torch.float64) * 0.5 - 1.0,
                    torch.rand(len(ts), B, 1, generator=g, dtype=torch.float64) * 2.0 - 4.0], -1)
    hps = {"nu": nu}
    r = fast_gp_mix.sample_posterior(x.to(cuda_device), y.to(cuda_device), ts, hps, 0, 0, seed=0, init=u0)
    r = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in r.items()}
    assert (r["diag"][..., DIAG["evals"]] == 1).all() and (r["diag"][..., DIAG["not_pd"]] == 0).all()
    assert torch.equal(r["log_samples"][:, :, 0], u0)
    assert torch.allclose(r["samples"][:, :, 0], torch.exp(u0), rtol=1e-15, atol=0)      # the device's exp
    xd, yd = x.double(), y.double()
    for i, t in enumerate(ts):
        for b in range(B):
            p = u0[i, b].clone().requires_grad_(True)
            U = M.potential_ref(xd[b, :t], yd[b, :t], p, hps, nu)
            (gr,) = torch.autograd.grad(U, p)
            Ud, gd = r["potential"][i, b].item(), r["grad"][i, b]
            assert abs(Ud - U.item()) <= 1e-9 * (1 + abs(U.item())), (t, b, Ud, U.item())
            assert (gd - gr).abs().max().item() <= 1e-7 * (1 + gr.norm().item()), (t, b, gd, gr)
            if t < T:   # latent predictive of row t at the same hyperparameters, mean 0
                th = torch.exp(u0[i, b])
                ls, s = th[:F], th[F]
                K = s * gp_matern_ref(xd[b, :t], xd[b, :t], ls, nu) + th[F + 1] * torch.eye(t, dtype=torch.float64)
                ks = s * gp_matern_ref(xd[b, :t], xd[b, t:t + 1], ls, nu)[:, 0]
                sol = torch.linalg.solve(K, torch.stack([yd[b, :t], ks], -1))
                mean, var = ks @ sol[:, 0], s - ks @ sol[:, 1]
                assert abs(r["mean"][i, b, 0].item() - mean.item()) <= 1e-9 * (1 + abs(mean.item()))
                assert abs(r["var"][i, b, 0].item() - var.item()) <= 1e-9 * (1 + abs(var.item()))
            else:
                assert math.isnan(r["mean"][i, b, 0].item())


def test_trajectories_follow_the_cpu_restatement(cuda_device):
    torch.manual_seed(21)
    B, T, F, W, S, seed = 8, 13, 1, 40, 10, 1234          # warmup 40: windows end at 5, 35, 39; 32 chains
    x, y, _ = fast_gp_mix.get_batch(B, T, F, device=cuda_device, batch_size_per_gp_sample=2)
    xb, yb = x.transpose(0, 1).contiguous(), y.transpose(0, 1).contiguous()
    ts = [3, 6, 9, 12]
    r = fast_gp_mix.sample_posterior(xb, yb, ts, {}, S, W, seed=seed, trace=True)
    tr = r["trace"].cpu().numpy()
    xd, yd = xb.double().cpu().numpy(), yb.double().cpu().numpy()
    agree, parted = 0, []
    for i, t in enumerate(ts):
        for b in range(B):
            c = M.nuts_chain(M.potential_and_grad_np(xd[b, :t], yd[b, :t]), F + 2, S, W, seed, b=b, t=t)
            du = np.abs(c["trace"][:, :F + 2] - tr[i, b, :, :F + 2]).max(1)
            same_depth = c["trace"][:, F + 3] == tr[i, b, :, F + 3]
            bad = np.nonzero((du > 1e-8) | ~same_depth)[0]
            if len(bad) == 0:
                agree += 1
            else:
                parted.append((t, b, int(bad[0]), float(du[bad[0]])))
    print(f"{agree} of {len(ts) * B} chains agree in all {W + S} iterations; parted (t, b, iteration, |du|): {parted}")
    assert agree >= 0.9 * len(ts) * B, parted


@pytest.mark.parametrize("os_conc", [0.5, 2.0])
def test_posterior_matches_quadrature(cuda_device, os_conc):
    torch.manual_seed(31 + int(10 * os_conc))
    hps = {"outputscale_concentration": os_conc}
    T, R = 61, 256
    x, y, _ = fast_gp_mix.get_batch(1, T, 1, device=cuda_device, hyperparameters=hps)
    xb = x.transpose(0, 1).repeat(R, 1, 1).contiguous()
    yb = y.transpose(0, 1).repeat(R, 1).contiguous()
    ts = [5, 20, 60]
    r = fast_gp_mix.sample_posterior(xb, yb, ts, hps, 100, 300, seed=77)
    xd, yd = xb[0].double().cpu(), yb[0].double().cpu()
    div = r["diag"][..., DIAG["div_sampling"]].sum().item()
    assert div < 0.01 * len(ts) * R * 100, div
    for i, t in enumerate(ts):
        q = M.quadrature_posterior(xd[:t], yd[:t], hps, x_star=xd[t, 0], y_star=yd[t], device=cuda_device)
        assert (q["edge_mass"] < 1e-6).all(), q
        u = r["log_samples"][i].cpu().numpy()                         # [R, S, 3]
        m = u.mean(1)
        v = (r["var"][i] + r["samples"][i, :, :, 2]).cpu().double()
        dens = torch.exp(-0.5 * (math.log(2 * math.pi) + torch.log(v) + (yd[t] - r["mean"][i].cpu()) ** 2 / v)).mean(1)
        for name, est, target in (("E[u]", m, q["mean"]), ("p(y_t)", dens.numpy()[:, None], np.asarray([q["pred"]]))):
            se = est.std(0, ddof=1) / math.sqrt(R)
            z = np.abs(est.mean(0) - target) / se
            print(f"t={t} os_conc={os_conc} {name}: chains {est.mean(0)} quadrature {target} se {se} z {z}")
            assert (z <= 5).all(), (t, name, est.mean(0), target, se)


def test_one_launch_equals_per_t_models_bitwise(cuda_device):
    torch.manual_seed(5)
    T, B, S, W = 12, 4, 20, 30
    x, y, _ = fast_gp_mix.get_batch(B, T, 2, device=cuda_device)
    ts = list(range(1, T))
    xb, yb = x.transpose(0, 1).contiguous(), y.transpose(0, 1).contiguous()
    r = fast_gp_mix.sample_posterior(xb, yb, ts, {}, S, W, seed=99)
    for i, t in enumerate(ts):
        model, likelihood = fast_gp_mix.get_mcmc_model(xb[:, :t], yb[:, :t], {}, cuda_device, S, W, seed=99)
        assert torch.equal(model.samples, r["samples"][i])
        pred = model(xb[:, t])                                        # [B, S, 1]
        assert torch.equal(pred.mean[..., 0], r["mean"][i]) and torch.equal(pred.variance[..., 0], r["var"][i])
        noisy = likelihood(pred)
        assert torch.equal(noisy.variance[..., 0], r["var"][i] + model.noise)
    # evaluate_ forms its losses from that same launch
    losses, _, all_losses = fast_gp_mix.evaluate_(x, y, y, {}, device=cuda_device, num_samples=S, warmup_steps=W, seed=99)
    for i, t in enumerate(ts):
        for b in range(B):
            l = -fast_gp_mix._mixture_logdensity(r["mean"][i, b], r["var"][i, b], y[t, b].double()).item()
            assert abs(all_losses[i][b] - l) <= 1e-12 * (1 + abs(l))
    again = fast_gp_mix.sample_posterior(xb, yb, ts, {}, S, W, seed=99)
    other = fast_gp_mix.sample_posterior(xb, yb, ts, {}, S, W, seed=100)
    assert torch.equal(again["samples"], r["samples"]) and torch.equal(again["diag"], r["diag"])
    assert not torch.equal(other["samples"], r["samples"])
    # the reference's single-dataset form: x [t, F], y [t]; predictive [S, m]
    model, _ = fast_gp_mix.get_mcmc_model(xb[0, :6], yb[0, :6], {}, cuda_device, S, W, seed=1)
    assert model(xb[0, 6:8]).mean.shape == (S, 2) and model.samples.shape == (1, S, 4)


def test_evaluate_follows_the_reference_conventions(cuda_device):
    torch.manual_seed(3)
    T, B, S, W = 10, 4, 20, 30
    x, y, _ = fast_gp_mix.get_batch(B, T, 1, device=cuda_device)
    losses, secs, all_losses = fast_gp_mix.evaluate_(x, y, y, {}, device=cuda_device, num_samples=S, warmup_steps=W,
                                                     seed=1)
    assert losses.shape == (T,) and losses[0] == 0 and losses.dtype == torch.float32 and secs > 0
    assert len(all_losses) == T - 1 and all(len(a) == B and isinstance(a[0], float) for a in all_losses)
    assert torch.allclose(losses[1:], torch.tensor([float(np.mean(a)) for a in all_losses]))
    part, _, part_all = fast_gp_mix.evaluate_(x, y, y, {}, device=cuda_device, num_samples=S, warmup_steps=W,
                                              min_seq_len=4, seed=1)
    assert part.shape == (T - 4,) and part_all == all_losses[3:]
    # full_range and use_likelihood against a torch.distributions restatement of get_mean_logdensity
    fr = (-3, 3)
    lfr, _, afr = fast_gp_mix.evaluate_(x, y, y, {}, device=cuda_device, num_samples=S, warmup_steps=W, seed=1,
                                        full_range=fr, use_likelihood=True)
    xb, yb = x.transpose(0, 1).contiguous(), y.transpose(0, 1).contiguous()
    r = fast_gp_mix.sample_posterior(xb, yb, list(range(1, T)), {}, S, W, seed=1)
    for i, t in enumerate([1, 5, 9]):
        for b in range(B):
            k = t - 1
            mean, var = r["mean"][k, b].cpu(), (r["var"][k, b] + r["samples"][k, b, :, 2]).cpu()
            dist = torch.distributions.Normal(mean, var.sqrt())
            w = 1. - (dist.cdf(torch.tensor(fr[0])) + (1. - dist.cdf(torch.tensor(fr[1]))))
            expect = -(torch.logsumexp(dist.log_prob(y[t, b].cpu().double()) - torch.log(w), 0) - math.log(S))
            assert abs(afr[k][b] - expect.item()) <= 1e-10 * (1 + abs(expect.item()))
    assert afr != all_losses
    with pytest.raises(ValueError, match="limit of 128"):
        fast_gp_mix.evaluate_(torch.rand(129, 2, 1), torch.randn(129, 2), None, {}, device=cuda_device)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        fast_gp_mix.evaluate_(x.cpu(), y.cpu(), None, {}, device="cpu")
    model, _ = fast_gp_mix.get_mcmc_model(xb[:, :5], yb[:, :5], {}, cuda_device, S, W, seed=2)
    assert model.diag.shape == (B, 6) and (model.diag[:, DIAG["leapfrog"]] > 0).all()
    assert model.step_size.shape == (B,) and (model.step_size > 0).all() and ((model.accept > 0) & (model.accept <= 1)).all()


def test_model_predicts_many_points_in_one_launch(cuda_device):
    torch.manual_seed(8)
    T, B, S, W, t = 16, 3, 10, 20, 9
    x, y, _ = fast_gp_mix.get_batch(B, T, 2, device=cuda_device)
    xb, yb = x.transpose(0, 1).contiguous(), y.transpose(0, 1).contiguous()
    model, _ = fast_gp_mix.get_mcmc_model(xb[:, :t], yb[:, :t], {}, cuda_device, S, W, seed=4)
    many = model(xb[:, t:])                                          # [B, S, T - t]
    assert many.mean.shape == (B, S, T - t) and (many.variance > 0).all()
    for j in range(T - t):                                           # the same factorisation, one row at a time
        one = model(xb[:, t + j])
        assert torch.equal(one.mean[..., 0], many.mean[..., j]) and torch.equal(one.variance[..., 0], many.variance[..., j])
    with pytest.raises(ValueError, match="limit of 128"):
        model(torch.rand(B, 128 - t + 1, 2, device=cuda_device))


def test_warmup_only_returns_the_last_state(cuda_device):
    """num_samples = 0 with warmup: the single output row is the state after the last warmup iteration, whatever the
    output buffers held, and the predictive is formed at it, bit for bit as an evaluate-only call there forms it."""
    torch.manual_seed(12)
    B, T, F, W, ts = 3, 12, 2, 25, [4, 9]
    x, y, _ = fast_gp_mix.get_batch(B, T, F, device=cuda_device)
    xb, yb = x.transpose(0, 1).contiguous(), y.transpose(0, 1).contiguous()
    r = fast_gp_mix.sample_posterior(xb, yb, ts, {}, 0, W, seed=6, max_tree_depth=4, trace=True, n_pred=2)
    assert r["samples"].shape == (len(ts), B, 1, F + 2) and r["trace"].shape == (len(ts), B, W, F + 4)
    assert torch.equal(r["log_samples"][:, :, 0], r["trace"][:, :, -1, :F + 2]) and torch.isnan(r["accept"]).all()
    e = fast_gp_mix.sample_posterior(xb, yb, ts, {}, 0, 0, init=r["log_samples"][:, :, 0], n_pred=2)
    for k in ("samples", "log_samples", "mean", "var"):
        assert torch.equal(e[k], r[k]), k
    assert torch.isfinite(r["mean"][:, :, 0]).all()

    kt, prior, _ = fast_gp_mix._fit_settings({})
    P, f64 = len(ts) * B, dict(dtype=torch.float64, device=cuda_device)

    def launch(fill):
        desc = L.gp_mcmc_desc(B, T, F, ts, kt, prior, 0, W, 6, 4, 2)
        out = {k: torch.full(shape, fill, **f64) for k, shape in
               (("samples", (P, 1, F + 2)), ("log_samples", (P, 1, F + 2)), ("mean", (P, 1, 2)), ("var", (P, 1, 2)),
                ("potential", (P,)), ("grad", (P, F + 2)), ("step_size", (P,)), ("accept", (P,)),
                ("trace", (P, W, F + 4)))}
        out["diag"] = torch.full((P, 6), -7, dtype=torch.int32, device=cuda_device)
        L.gp_mcmc(xb.float(), yb.float(), desc, out["samples"], out["step_size"], out["accept"], out["diag"],
                  **{k: v for k, v in out.items() if k not in ("samples", "step_size", "accept", "diag")})
        return out

    a, b = launch(float("nan")), launch(0.0)
    for k in a:
        assert torch.equal(a[k].isnan(), b[k].isnan()) and torch.equal(a[k].nan_to_num(0.0), b[k].nan_to_num(0.0)), k
        assert k == "accept" or not a[k].isnan().any(), k
    assert torch.equal(a["log_samples"].view(len(ts), B, 1, F + 2), r["log_samples"])


def test_a_chain_without_a_finite_start_is_not_run(cuda_device):
    B, T, F = 2, 8, 1
    x = torch.full((B, T, F), 0.5, device=cuda_device)              # identical rows: K = s 11^T + noise I
    y = torch.randn(B, T, device=cuda_device)
    u0 = torch.zeros(1, B, F + 2, dtype=torch.float64)
    u0[0, 0, F + 1] = -1000.0                                        # noise exp(-1000) = 0: K is singular in dataset 0
    r = fast_gp_mix.sample_posterior(x, y, [6], {}, 5, 10, seed=3, init=u0, trace=True)
    assert torch.isnan(r["samples"][0, 0]).all() and torch.isnan(r["log_samples"][0, 0]).all()
    assert torch.isnan(r["mean"][0, 0]).all() and torch.isnan(r["trace"][0, 0]).all()
    assert r["potential"][0, 0].item() == math.inf and math.isnan(r["step_size"][0, 0].item())
    assert r["diag"][0, 0, DIAG["not_pd"]].item() == 1 and r["diag"][0, 0, DIAG["leapfrog"]].item() == 0
    assert torch.isfinite(r["samples"][0, 1]).all() and r["diag"][0, 1, DIAG["leapfrog"]].item() > 0
    # evaluate-only at the same point reports U = +inf and the NaN predictive of a non-PD matrix
    e = fast_gp_mix.sample_posterior(x, y, [6], {}, 0, 0, seed=3, init=u0)
    assert e["potential"][0, 0].item() == math.inf and math.isnan(e["mean"][0, 0, 0].item())
    assert math.isfinite(e["potential"][0, 1].item())
