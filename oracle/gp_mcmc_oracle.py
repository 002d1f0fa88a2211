"""CPU oracle of the fully Bayesian GP baseline -- TEST INFRASTRUCTURE ONLY (plain torch / numpy / Python floats, sharing
no code with the CUDA engine; only tests/ and tools/ import it).

Restates reference priors/fast_gp_mix.py:171-268 (pyro 1.7 NUTS over the Gamma hyperpriors of botorch's SingleTaskGP,
constant mean fixed at 0) on the posterior p(u | y[:t]), u = log(ls_1..F, s, noise):
  * `potential_ref` / `potential_and_grad_np`: U(u) = -log N(y | 0, K) - sum_k log Gamma(theta_k) - sum_k u_k and its
    gradient (fp64 torch with autograd, and a closed-form numpy version for the CPU chains);
  * `Rng`: the counter-based random numbers of csrc/counter_rng.cuh and the kernel's Box-Muller transform;
  * `nuts_chain`: the sampler itself, with the kernel's algorithm, constants, operation order and random-number keys
    (it is the written contract of csrc/gp_mcmc.cu; PARITY WITH PYRO UNPINNED: pyro is not installed);
  * `quadrature_posterior`: a tensor-product grid over u for F = 1 (d = 3) giving E[u_k], Var[u_k] and the exact mixture
    predictive density of a new observation.
"""
import math

import numpy as np
import torch

from oracle.gp_fit_oracle import _gamma_logpdf, _gp_fit_priors, gp_matern_ref

# ---------------------------------------------------------------------------------------------------------- potential


def potential_ref(x, y, u, hps=None, nu=2.5):
    """U(u) for ONE problem, fp64 torch (differentiable): x [t,F], y [t], u [F+2]."""
    t, F = x.shape
    la, lb, oa, ob, na, nb = _gp_fit_priors(hps)
    theta = torch.exp(u)
    ls, s, noise = theta[:F], theta[F], theta[F + 1]
    K = s * gp_matern_ref(x, x, ls, nu) + noise * torch.eye(t, dtype=x.dtype)
    Lc = torch.linalg.cholesky(K)
    alpha = torch.cholesky_solve(y.unsqueeze(-1), Lc)
    logn = -0.5 * (y.unsqueeze(-1) * alpha).sum() - torch.log(torch.diagonal(Lc)).sum() - 0.5 * t * math.log(2 * math.pi)
    lp = _gamma_logpdf(ls, la, lb).sum() + _gamma_logpdf(s, oa, ob) + _gamma_logpdf(noise, na, nb) + u.sum()
    return -(logn + lp)


def potential_value_and_grad_ref(x, y, u, hps=None, nu=2.5):
    """(U, dU/du) as float / numpy through autograd; (+inf, zeros) where K is not positive definite."""
    p = torch.as_tensor(np.asarray(u, dtype=np.float64)).clone().requires_grad_(True)
    try:
        U = potential_ref(x, y, p, hps, nu)
    except torch.linalg.LinAlgError:
        return float("inf"), np.zeros(p.numel())
    (g,) = torch.autograd.grad(U, p)
    return float(U.detach()), g.numpy()


def _matern_np(r2, nu):
    """k(r) and g(r) = -k'(r)/r from r^2 (numpy, elementwise)."""
    r = np.sqrt(r2)
    if nu == 0.5:
        e = np.exp(-r)
        with np.errstate(divide="ignore", invalid="ignore"):
            return e, np.where(r > 0, e / np.where(r > 0, r, 1.0), 0.0)
    if nu == 1.5:
        a = math.sqrt(3.0) * r
        e = np.exp(-a)
        return (1 + a) * e, 3.0 * e
    a = math.sqrt(5.0) * r
    e = np.exp(-a)
    return (1 + a + 5.0 / 3.0 * r2) * e, 5.0 / 3.0 * (1 + a) * e


def potential_and_grad_np(x, y, hps=None, nu=2.5):
    """A closed-form numpy potential for ONE problem (x [t,F], y [t] float64 arrays) for the CPU chains: returns
    f(u) -> (U, grad list)."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    t, F = x.shape
    la, lb, oa, ob, na, nb = _gp_fit_priors(hps)
    const = [a * math.log(b) - math.lgamma(a) for a, b in ((la, lb),) * F + ((oa, ob), (na, nb))]
    conc = [la] * F + [oa, na]
    rate = [lb] * F + [ob, nb]
    D2 = (x[:, None, :] - x[None, :, :]) ** 2                  # [t, t, F]

    def f(u):
        u = np.asarray(u, np.float64)
        th = np.exp(u)
        ls, s, noise = th[:F], th[F], th[F + 1]
        r2 = (D2 / ls ** 2).sum(-1)
        k, g = _matern_np(r2, nu)
        K = s * k + noise * np.eye(t)
        try:
            Lc = np.linalg.cholesky(K)
        except np.linalg.LinAlgError:
            return float("inf"), [0.0] * (F + 2)
        Li = np.linalg.inv(Lc)
        Kinv = Li.T @ Li
        alpha = Kinv @ y
        logn = -0.5 * y @ alpha - np.log(np.diag(Lc)).sum() - 0.5 * t * math.log(2 * math.pi)
        lp = sum(c + a * ui - b * ti for c, a, b, ui, ti in zip(const, conc, rate, u, th))
        W = np.outer(alpha, alpha) - Kinv
        grad = [-(0.5 * s / ls[d] ** 2 * (W * g * D2[:, :, d]).sum()) - la + lb * ls[d] for d in range(F)]
        grad.append(-(0.5 * s * (W * k).sum()) - oa + ob * s)
        grad.append(-(0.5 * noise * np.trace(W)) - na + nb * noise)
        U = -(logn + lp)
        return (float(U) if U == U else float("inf")), [float(v) for v in grad]
    return f


# ---------------------------------------------------------------------------------------------------------- random numbers
M32 = 0xFFFFFFFF


def mix32(x):
    x ^= x >> 16
    x = (x * 0x7FEB352D) & M32
    x ^= x >> 15
    x = (x * 0x846CA68B) & M32
    x ^= x >> 16
    return x


def hash5(seed, tag, a, b, c):
    h = mix32(seed ^ ((tag * 0x9E3779B1) & M32))
    h = mix32(h ^ ((a * 0x85EBCA77) & M32))
    h = mix32(h ^ ((b * 0xC2B2AE3D) & M32))
    return mix32(h ^ ((c * 0x27D4EB2F) & M32))


def uniform_double(hi, lo):
    return ((hi >> 5) * 67108864.0 + (lo >> 6)) * (1.0 / 9007199254740992.0)


class Rng:
    """Draw k of iteration key `it` = uniform_double(hash5(seed, b, t, it, 2k), hash5(seed, b, t, it, 2k + 1))."""

    def __init__(self, seed, b, t):
        self.seed, self.b, self.t, self.it, self.ctr = int(seed) & M32, int(b) & M32, int(t) & M32, 0, 0

    def key(self, it):
        self.it, self.ctr = int(it) & M32, 0

    def uniform(self):
        k = self.ctr
        self.ctr += 1
        return uniform_double(hash5(self.seed, self.b, self.t, self.it, (2 * k) & M32),
                              hash5(self.seed, self.b, self.t, self.it, (2 * k + 1) & M32))

    def normal(self):
        u1 = 1.0 - self.uniform()
        u2 = self.uniform()
        return math.sqrt(-2.0 * math.log(u1)) * math.cos(6.283185307179586 * u2)


# ---------------------------------------------------------------------------------------------------------- NUTS
TARGET_ACCEPT, DA_GAMMA, DA_T0, DA_KAPPA = 0.8, 0.05, 10.0, 0.75
MAX_ENERGY_ERROR = 1000.0
LOG_ACCEPT_THRESHOLD = -0.2231435513142097
SEARCH_MAX, INIT_TRIES = 100, 100
INF = float("inf")


def adaptation_windows(W):
    """End index of every warmup window (pyro WarmupAdapter._build_adaptation_schedule)."""
    if W < 20:
        return [W - 1]
    start_buf, end_buf, init_win = 75, 50, 25
    if start_buf + end_buf + init_win > W:
        start_buf, end_buf = int(0.15 * W), int(0.1 * W)
        init_win = W - start_buf - end_buf
    ends = [start_buf - 1]
    end_start = W - end_buf
    next_size, next_start = init_win, start_buf
    while next_start < end_start:
        cur_start, cur_size = next_start, next_size
        if 3 * cur_size <= end_start - cur_start:
            next_size = 2 * cur_size
        else:
            cur_size = end_start - cur_start
        next_start = cur_start + cur_size
        ends.append(next_start - 1)
    ends.append(W - 1)
    return ends


def _logaddexp(x, y):
    mn, mx = (x, y) if x < y else (y, x)
    return math.log1p(math.exp(mn - mx)) + mx


def _kinetic(w):
    e = 0.0
    for v in w:
        e = e + v * v
    return 0.5 * e


def _is_turning(wl, wr, wsum):
    left = right = 0.0
    for a, b, s in zip(wl, wr, wsum):
        rho = s - (a + b) / 2.0
        left = left + a * rho
        right = right + b * rho
    return left <= 0.0 or right <= 0.0


def _exp(v):
    try:
        return math.exp(v)
    except OverflowError:
        return INF


def nuts_chain(pot, d, num_samples, warmup_steps, seed, b=0, t=0, init=None, max_tree_depth=10):
    """One NUTS chain on the potential pot(u) -> (U, grad) in d dimensions, with the kernel's algorithm and random keys
    (dataset b, prefix t).  Returns a dict: samples [S, d] (u), trace [W+S, d+2] (u, step size used, tree depth),
    step_size, accept, diag (the kernel's six counters), potential, grad."""
    W, S = int(warmup_steps), int(num_samples)
    rng = Rng(seed, b, t)
    diag = {"leapfrog": 0, "evals": 0, "div_warmup": 0, "div_sampling": 0, "max_depth_hits": 0, "not_pd": 0}

    def evaluate(u):
        U, g = pot(u)
        diag["evals"] += 1
        if not U < INF:
            diag["not_pd"] += 1
            return INF, [0.0] * d
        return U, list(g)

    inv_m = [1.0] * d
    sqrt_im = [1.0] * d
    rsqrt_im = [1.0] * d

    def set_inv_mass(vals):
        for i, v in enumerate(vals):
            inv_m[i], sqrt_im[i], rsqrt_im[i] = v, math.sqrt(v), 1.0 / math.sqrt(v)

    def draw_momentum():
        w = [rng.normal() for _ in range(d)]
        return [w[i] * rsqrt_im[i] for i in range(d)], w, _kinetic(w)

    def leapfrog(z, r, g, e):
        h = 0.5 * e
        rh = [r[i] + h * (-g[i]) for i in range(d)]
        zn = [z[i] + e * (inv_m[i] * rh[i]) for i in range(d)]
        U, gn = evaluate(zn)
        rn = [rh[i] + h * (-gn[i]) for i in range(d)]
        wn = [rn[i] * sqrt_im[i] for i in range(d)]
        en = U + _kinetic(wn)
        return zn, rn, gn, U, wn, (en if en == en else INF)

    # ---- initial point
    rng.key(0)
    for attempt in range(INIT_TRIES):
        z = list(init) if init is not None else [-2.0 + 4.0 * rng.uniform() for _ in range(d)]
        pe, g = evaluate(z)
        if init is not None or pe < INF:
            break
    out = {"diag": diag}
    if W == 0 and S == 0:
        out.update(samples=np.asarray([z]), trace=np.zeros((0, d + 2)), step_size=0.0, accept=float("nan"),
                   potential=pe, grad=np.asarray(g))
        return out
    state = {"eps": 1.0, "center": 0.0, "x": 0.0, "xavg": 0.0, "gavg": 0.0, "t": 0}

    def search():                                           # pyro HMC._find_reasonable_step_size
        eps, first, count, s_dir, scale = state["eps"], True, 0, 0, 1.0
        while True:
            if not first:
                eps = scale * eps
            r, w, ke = draw_momentum()
            e0 = ke + pe
            _, _, _, _, _, en = leapfrog(z, r, g, eps)
            delta = en - e0
            nd = 1 if LOG_ACCEPT_THRESHOLD < -delta else -1
            if first:
                first, s_dir, scale = False, nd, (2.0 if nd == 1 else 0.5)
                continue
            if nd != s_dir:
                break
            count += 1
            if not count < SEARCH_MAX:
                break
        state.update(eps=eps, center=math.log(10.0 * eps), xavg=0.0, gavg=0.0, t=0)

    search()
    ends = adaptation_windows(W)
    cw = 0
    wf_n, wf_mean, wf_m2 = 0, [0.0] * d, [0.0] * d
    samples, trace, acc_sampling = [], [], 0.0
    for it in range(W + S):
        rng.key(it + 1)
        eps = state["eps"]
        r0, w0, ke = draw_momentum()
        energy0 = ke + pe
        ez, er, eg, ew = [list(z), list(z)], [list(r0), list(r0)], [list(g), list(g)], [list(w0), list(w0)]
        w_sum, weight, acc_sum, n_prop, depth = list(w0), 0.0, 0.0, 0, 0
        while True:
            s = 1 if rng.uniform() < 0.5 else 0
            e = eps if s else -eps
            stack, sub_acc, sub_n, status = [None] * (depth + 1), 0.0, 0, 1
            for leaf in range(1 << depth):
                zn, rn, gn, U, wn, en = leapfrog(ez[s], er[s], eg[s], e)
                diag["leapfrog"] += 1
                ez[s], er[s], eg[s], ew[s] = zn, rn, gn, wn
                sliced = en + (-energy0)
                acc = _exp(-(en - energy0))
                sub_acc = sub_acc + (acc if acc < 1.0 else 1.0)
                sub_n += 1
                if sliced > MAX_ENERGY_ERROR:
                    status = 3
                    break
                C = {"wf": wn, "wl": wn, "ws": list(wn), "z": zn, "g": gn, "pe": U, "weight": -sliced}
                lvl = 0
                while (leaf >> lvl) & 1:
                    H = stack[lvl]
                    wt = _logaddexp(H["weight"], C["weight"])
                    p_other = _exp(C["weight"] - wt)
                    if not rng.uniform() < p_other:
                        C["z"], C["g"], C["pe"] = H["z"], H["g"], H["pe"]
                    C["weight"] = wt
                    C["ws"] = [H["ws"][i] + C["ws"][i] for i in range(d)]
                    C["wf"] = H["wf"]
                    if _is_turning(C["wf"], C["wl"], C["ws"]):
                        status = 2
                        break
                    lvl += 1
                if status == 2:
                    break
                stack[lvl] = C
            acc_sum = acc_sum + sub_acc
            n_prop += sub_n
            if status == 3:
                diag["div_warmup" if it < W else "div_sampling"] += 1
                break
            if status == 2:
                break
            depth += 1
            if rng.uniform() < _exp(C["weight"] - weight):
                z, g, pe = list(C["z"]), list(C["g"]), C["pe"]
            w_sum = [w_sum[i] + C["ws"][i] for i in range(d)]
            if _is_turning(ew[0], ew[1], w_sum):
                break
            weight = _logaddexp(weight, C["weight"])
            if depth >= max_tree_depth:
                diag["max_depth_hits"] += 1
                break
        accept_prob = acc_sum / n_prop
        trace.append(list(z) + [eps, float(depth)])
        if it >= W:
            samples.append(list(z))
            acc_sampling = acc_sampling + accept_prob
            continue
        tp = it + 1                                         # pyro WarmupAdapter.step(t = it + 1)
        if tp >= W:
            continue
        mm = 0 < cw < len(ends) - 1
        state["t"] += 1
        tt = state["t"] + DA_T0
        state["gavg"] = (1.0 - 1.0 / tt) * state["gavg"] + (TARGET_ACCEPT - accept_prob) / tt
        state["x"] = state["center"] - math.sqrt(float(state["t"])) / DA_GAMMA * state["gavg"]
        wt = math.pow(float(state["t"]), -DA_KAPPA)
        state["xavg"] = (1.0 - wt) * state["xavg"] + wt * state["x"]
        state["eps"] = math.exp(state["x"])
        if mm:
            wf_n += 1
            for i in range(d):
                pre = z[i] - wf_mean[i]
                wf_mean[i] = wf_mean[i] + pre / wf_n
                wf_m2[i] = wf_m2[i] + pre * (z[i] - wf_mean[i])
        if tp != ends[cw]:
            continue
        if cw == len(ends) - 1:
            cw += 1
            state["eps"] = math.exp(state["xavg"])
            continue
        if cw == 0:
            cw += 1
            continue
        n = float(wf_n)
        set_inv_mass([(n / (n + 5.0)) * (wf_m2[i] / (n - 1.0)) + 1e-3 * (5.0 / (n + 5.0)) for i in range(d)])
        wf_n, wf_mean, wf_m2 = 0, [0.0] * d, [0.0] * d
        cw += 1
        search()
    out.update(samples=np.asarray(samples).reshape(S, d), trace=np.asarray(trace), step_size=state["eps"],
               accept=acc_sampling / S if S else float("nan"), potential=pe, grad=np.asarray(g))
    return out


def gaussian_potential(scales):
    """Potential of a centred Gaussian with independent coordinates of the given scales."""
    inv = [1.0 / (s * s) for s in scales]

    def f(u):
        return 0.5 * sum(v * v * a for v, a in zip(u, inv)), [v * a for v, a in zip(u, inv)]
    return f


def gaussian_chain_job(args):
    """nuts_chain on gaussian_potential(scales) for chain (dataset slot) b: a unit of work of a process pool."""
    scales, num_samples, warmup_steps, seed, b = args
    return nuts_chain(gaussian_potential(scales), len(scales), num_samples, warmup_steps, seed, b=b)["samples"]


def gp_chain_job(args):
    """nuts_chain on the numpy GP potential of (x, y) for dataset slot b: a unit of work of a process pool."""
    x, y, hps, nu, num_samples, warmup_steps, seed, b = args
    pot = potential_and_grad_np(x, y, hps, nu)
    return nuts_chain(pot, np.asarray(x).shape[1] + 2, num_samples, warmup_steps, seed, b=b, t=len(y))["samples"]


# ---------------------------------------------------------------------------------------------------------- quadrature
def _grid_logpost(x, y, U, hps, nu, x_star, y_star, chunk, device):
    """log of the unnormalised posterior at grid points U [G, 3] (F = 1) and, with x_star / y_star, the log predictive
    density of y_star (observation noise included) at every point."""
    t = x.shape[0]
    la, lb, oa, ob, na, nb = _gp_fit_priors(hps)
    out_lp, out_pred = [], []
    x = x.to(device, torch.float64)
    y = y.to(device, torch.float64)
    for i in range(0, U.shape[0], chunk):
        u = U[i:i + chunk].to(device)
        th = torch.exp(u)
        ls, s, noise = th[:, 0], th[:, 1], th[:, 2]
        lp = (_gamma_logpdf(ls, la, lb) + _gamma_logpdf(s, oa, ob) + _gamma_logpdf(noise, na, nb) + u.sum(1))
        if t > 0:
            d2 = ((x[:, None, 0] - x[None, :, 0]) ** 2)[None] / ls[:, None, None] ** 2
            k = _matern_t(d2, nu)
            K = s[:, None, None] * k + noise[:, None, None] * torch.eye(t, dtype=torch.float64, device=device)
            Lc, info = torch.linalg.cholesky_ex(K)
            alpha = torch.cholesky_solve(y[None, :, None].expand(len(u), t, 1), Lc)
            logn = (-0.5 * (y[None, :] * alpha[..., 0]).sum(1) - torch.log(torch.diagonal(Lc, dim1=1, dim2=2)).sum(1)
                    - 0.5 * t * math.log(2 * math.pi))
            lp = torch.where(info == 0, lp + logn, torch.full_like(lp, -math.inf))
        out_lp.append(lp)
        if x_star is not None:
            xs = torch.as_tensor(float(x_star), dtype=torch.float64, device=device)
            if t > 0:
                ks = s[:, None] * _matern_t(((x[None, :, 0] - xs) ** 2) / ls[:, None] ** 2, nu)
                sol = torch.cholesky_solve(ks[..., None], Lc)[..., 0]
                mean = (ks * alpha[..., 0]).sum(1)
                var = s - (ks * sol).sum(1) + noise
            else:
                mean, var = torch.zeros_like(s), s + noise
            out_pred.append(-0.5 * (math.log(2 * math.pi) + torch.log(var) + (float(y_star) - mean) ** 2 / var))
    return torch.cat(out_lp), (torch.cat(out_pred) if out_pred else None)


def _matern_t(r2, nu):
    r = r2.clamp_min(0).sqrt()
    if nu == 0.5:
        return torch.exp(-r)
    if nu == 1.5:
        a = math.sqrt(3.0) * r
        return (1 + a) * torch.exp(-a)
    a = math.sqrt(5.0) * r
    return (1 + a + 5.0 / 3.0 * r2) * torch.exp(-a)


def quadrature_posterior(x, y, hps=None, nu=2.5, x_star=None, y_star=None, n=128, box=((-80., 12.),) * 3,
                         device="cpu", chunk=8192):
    """Posterior moments of u = (log ls, log s, log noise) for F = 1 on a tensor-product grid: x [t,1], y [t] (t may be
    0).  A coarse pass over `box` locates the mass; the final grid (n points per axis) covers where the coarse marginals
    exceed 1e-14 of their peak, one coarse step wider.  Returns dict mean [3], var [3], edge_mass [3] (largest marginal
    mass of a boundary slab of the final grid) and, with x_star / y_star, pred = p(y_star | y) with the noise included."""
    x = torch.as_tensor(x, dtype=torch.float64).reshape(-1, 1)
    y = torch.as_tensor(y, dtype=torch.float64).reshape(-1)

    def grid(lo_hi, m):
        axes = [torch.linspace(lo, hi, m, dtype=torch.float64) for lo, hi in lo_hi]
        return axes, torch.stack(torch.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)

    nc = 64
    axes, U = grid(box, nc)
    lp, _ = _grid_logpost(x, y, U, hps, nu, None, None, chunk, device)
    w = torch.softmax(lp.cpu(), 0).reshape(nc, nc, nc)
    new_box = []
    for k in range(3):
        marg = w.sum(dim=tuple(j for j in range(3) if j != k))
        keep = torch.nonzero(marg > 1e-14 * marg.max())[:, 0]
        step = float(axes[k][1] - axes[k][0])
        new_box.append((float(axes[k][keep.min()]) - step, float(axes[k][keep.max()]) + step))
    axes, U = grid(new_box, n)
    lp, lpred = _grid_logpost(x, y, U, hps, nu, x_star, y_star, chunk, device)
    lp = lp.cpu()
    w = torch.softmax(lp, 0)
    mean = (w[:, None] * U).sum(0)
    var = (w[:, None] * (U - mean) ** 2).sum(0)
    w3 = w.reshape(n, n, n)
    edge = []
    for k in range(3):
        marg = w3.sum(dim=tuple(j for j in range(3) if j != k))
        edge.append(float(max(marg[0], marg[-1])))
    out = {"mean": mean.numpy(), "var": var.numpy(), "edge_mass": np.asarray(edge), "box": new_box}
    if lpred is not None:
        out["pred"] = float(torch.exp(torch.logsumexp(lp + lpred.cpu(), 0) - torch.logsumexp(lp, 0)))
    return out
