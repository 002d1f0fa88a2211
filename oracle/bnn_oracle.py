"""CPU oracle of the Bayesian-NN prior and its NUTS baseline -- TEST INFRASTRUCTURE ONLY (plain torch / numpy, sharing no
code with the CUDA engine; only tests/ and tools/ import it).

Restates reference mcmc_svi_transformer_on_bayesian.py:28-67 (BayesianModel: fc1 [E, F] and fc2 [2, E] with N(0, 1) weights
and biases, `nn.Sequential(fc1, fc2)` with no nonlinearity, a Categorical observation on the softmax) and
priors/pyro.py:10-34 (one model call per dataset, x standardised over the sequence axis):
  * `potential_ref` / `potential_and_grad_np`: U(theta) = 1/2 |theta|^2 + d/2 log 2 pi - sum_r log softmax(logits_r)[y_r]
    for theta = (W1, b1, W2, b2) flattened in that order, in fp64 torch (gradient by autograd) and in closed-form numpy
    for `gp_mcmc_oracle.nuts_chain`, which is generic in the potential and is the written contract of csrc/bnn_mcmc.cu
    (PARITY WITH PYRO UNPINNED: pyro is not installed);
  * `prior_forward_ref`: the prior's class probabilities, class decisions and standardised x in fp64 from given weights,
    inputs and uniforms;
  * `importance_predictive`: the posterior predictive p(y* = 1 | x*, D) = E[p(y* | theta) p(D | theta)] / E[p(D | theta)]
    over theta ~ prior by self-normalised importance sampling, with its standard error (small n only: the weights
    degenerate as the likelihood sharpens).
"""
import math

import numpy as np
import torch

from oracle.gp_mcmc_oracle import nuts_chain

HALF_LOG_2PI = 0.5 * math.log(2 * math.pi)


def dim(F, E):
    return E * F + 3 * E + 2


def unpack(theta, F, E):
    """theta [..., d] -> W1 [..., E, F], b1 [..., E], W2 [..., 2, E], b2 [..., 2] (views)."""
    lead = theta.shape[:-1]
    o = E * F
    return (theta[..., :o].reshape(*lead, E, F), theta[..., o:o + E], theta[..., o + E:o + 3 * E].reshape(*lead, 2, E),
            theta[..., o + 3 * E:])


def logits_ref(theta, x, F, E):
    """Logits [..., n, 2] of rows x [n, F] under theta [..., d] (torch)."""
    W1, b1, W2, b2 = unpack(theta, F, E)
    h = x @ W1.transpose(-1, -2) + b1.unsqueeze(-2)
    return h @ W2.transpose(-1, -2) + b2.unsqueeze(-2)


def potential_ref(x, y, theta, F, E):
    """U(theta) for ONE dataset, fp64 torch (differentiable): x [n, F], y [n] (0 / 1), theta [d]."""
    lp = torch.log_softmax(logits_ref(theta, x, F, E), -1)
    nll = -lp.gather(-1, y.long().unsqueeze(-1)).sum()
    return 0.5 * (theta * theta).sum() + theta.numel() * HALF_LOG_2PI + nll


def potential_value_and_grad_ref(x, y, theta, F, E):
    p = torch.as_tensor(np.asarray(theta, dtype=np.float64)).clone().requires_grad_(True)
    U = potential_ref(x, y, p, F, E)
    (g,) = torch.autograd.grad(U, p)
    return float(U.detach()), g.numpy()


def potential_and_grad_np(x, y, F, E):
    """A closed-form numpy potential for ONE dataset (x [n, F] float64, y [n] 0 / 1) for the CPU chains: returns
    f(theta) -> (U, grad list), with the backward written out: dl = p - onehot, dW2 = dl^T h, dh = dl W2, dW1 = dh^T x."""
    x = np.asarray(x, np.float64)
    yi = np.asarray(y).astype(np.int64)
    n = x.shape[0]
    onehot = np.zeros((n, 2))
    onehot[np.arange(n), yi] = 1.0
    d = dim(F, E)

    def f(theta):
        th = np.asarray(theta, np.float64)
        W1, b1, W2, b2 = unpack(th, F, E)
        h = x @ W1.T + b1
        l = h @ W2.T + b2
        m = l.max(1)
        with np.errstate(over="ignore", invalid="ignore"):
            lse = m + np.log(np.exp(l[:, 0] - m) + np.exp(l[:, 1] - m))
            nll = lse - l[np.arange(n), yi]
            dl = np.exp(l - lse[:, None]) - onehot
            dh = dl @ W2
            grad = th + np.concatenate([(dh.T @ x).ravel(), dh.sum(0), (dl.T @ h).ravel(), dl.sum(0)])
            U = (0.5 * float(th @ th) + d * HALF_LOG_2PI) + float(nll.sum())
        return (U if U == U else float("inf")), [float(v) for v in grad]
    return f


def bnn_chain_job(args):
    """nuts_chain on the numpy potential of (x, y) for dataset slot b: a unit of work of a process pool.  Returns the
    chain's dict (samples [S, d], trace [W + S, d + 2], diag, ...)."""
    x, y, F, E, num_samples, warmup_steps, seed, b, max_tree_depth = args
    return nuts_chain(potential_and_grad_np(x, y, F, E), dim(F, E), num_samples, warmup_steps, seed, b=b, t=len(y),
                      max_tree_depth=max_tree_depth)


def predictive_ref(theta, x_test, F, E):
    """Class-1 probability [..., n_test] of rows x_test [n_test, F] under theta [..., d] (torch fp64)."""
    return torch.softmax(logits_ref(theta, x_test, F, E), -1)[..., 1]


def prior_forward_ref(weights, x_raw, u, F, E):
    """The prior's forward in fp64 from the drawn values: weights [B, d], x_raw [T, B, F], u [T, B].  Returns
    (p0 [T, B] the class-0 probability, y [T, B] = 0 where u < p0 else 1, x [T, B, F] standardised over the sequence axis
    as priors/pyro.py:20-25 normalize_data does)."""
    w, xr, u = weights.double(), x_raw.double(), u.double()
    l = logits_ref(w, xr.transpose(0, 1), F, E)                  # [B, T, 2]
    p0 = torch.softmax(l, -1)[..., 0].transpose(0, 1)
    y = (~(u < p0)).double()
    xn = (xr - xr.mean(0)) / (xr.std(0) + .000001)
    return p0, y, xn


def importance_predictive(x_train, y_train, x_test, F, E, num_draws=1 << 20, chunk=1 << 18, seed=0, device="cpu"):
    """Self-normalised importance sampling of the posterior predictive with the prior as the proposal: theta_k ~ N(0, I),
    w_k = p(D | theta_k), estimate sum_k w_k p(y* = 1 | x*, theta_k) / sum_k w_k per test row.  x_train [n, F], y_train [n],
    x_test [m, F].  Returns dict p1 [m], se [m] (delta-method standard error of the ratio) and ess (effective sample
    size of the weights)."""
    dev = torch.device(device)
    xt = torch.as_tensor(x_train, dtype=torch.float64, device=dev)
    yt = torch.as_tensor(y_train, device=dev).long()
    xs = torch.as_tensor(x_test, dtype=torch.float64, device=dev)
    g = torch.Generator().manual_seed(seed)
    logw, p1 = [], []
    for i in range(0, num_draws, chunk):
        th = torch.randn(min(chunk, num_draws - i), dim(F, E), generator=g, dtype=torch.float64).to(dev)
        lp = torch.log_softmax(logits_ref(th, xt, F, E), -1)      # [K, n, 2]
        logw.append(lp.gather(-1, yt.expand(th.shape[0], -1).unsqueeze(-1)).squeeze(-1).sum(-1))
        p1.append(predictive_ref(th, xs, F, E))
    logw, p1 = torch.cat(logw), torch.cat(p1)
    w = torch.softmax(logw, 0)                                    # normalised weights
    est = (w[:, None] * p1).sum(0)
    se = torch.sqrt((w[:, None] ** 2 * (p1 - est) ** 2).sum(0))
    return {"p1": est.cpu().numpy(), "se": se.cpu().numpy(), "ess": float(1.0 / (w * w).sum())}
