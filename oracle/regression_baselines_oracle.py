"""fp64 numpy restatement of csrc/regression_baselines.cu (the ridge baseline and the exact GP of priors.gp), with the
per-element error bounds the tests hold the kernels to.  TEST INFRASTRUCTURE ONLY.

Each function takes one dataset: x [T, F], y / target [T] (any float dtype; the kernels read fp32).
"""
import numpy as np

EPS = np.finfo(np.float64).eps
ALPHA_GP = 1e-10
LOG_2PI = float(np.log(2 * np.pi))


# ------------------------------------------------------------------------------------------------ ridge
def ridge_prefix_ref(x, y, target, alpha):
    """pred, sq_err [T] (index 0 NaN) and per prefix the quantities of ridge_bound: Ridge(alpha) with intercept on rows < t
    predicts row t.  Minimum-norm solution for alpha = 0, singular values of the centred rows at or below
    max(t, F) eps s_max dropped; every singular value used for alpha > 0."""
    x, y, target = (np.asarray(v, dtype=np.float64) for v in (x, y, target))
    T, F = x.shape
    pred, sq = np.full(T, np.nan), np.full(T, np.nan)
    info = [None]
    for t in range(1, T):
        mx, my = x[:t].mean(0), y[:t].mean()
        Xc, yc = x[:t] - mx, y[:t] - my
        U, s, Vt = np.linalg.svd(Xc, full_matrices=False)
        smax = s.max() if s.size else 0.0
        keep = s > 0 if alpha > 0 else s > max(t, F) * EPS * smax
        coef = np.where(keep, s / np.where(keep, s * s + alpha, 1.0), 0.0)
        w = Vt.T @ (coef * (U.T @ yc))
        dx = x[t] - mx
        pred[t] = my + dx @ w
        sq[t] = (target[t] - pred[t]) ** 2
        sk = s[keep]
        kappa = (smax ** 2 + alpha) / (sk.min() ** 2 + alpha) if sk.size else 1.0
        info.append(dict(my=abs(my), dx=np.linalg.norm(dx), w=np.linalg.norm(w), res=np.linalg.norm(yc - Xc @ w),
                         smax=smax, kappa=kappa, t=t, F=F))
    return pred, sq, info


def ridge_bound(info):
    """Per-element bound on |pred_device - pred_ref| from the perturbation of a least-squares / ridge solution whose data
    carry relative errors of O((t + F) eps): both sides' errors, kappa the condition of the normal matrix over the kept
    singular values."""
    b = np.full(len(info), np.nan)
    for t, d in enumerate(info):
        if d is None:
            continue
        g = 16.0 * (d["t"] + d["F"]) * EPS
        b[t] = g * (d["my"] + d["dx"] * d["w"] * (1.0 + d["kappa"])
                    + d["dx"] * d["kappa"] * d["res"] / max(np.sqrt(d["smax"] ** 2), 1e-300)) + 1e-300
    return b


# ------------------------------------------------------------------------------------------------ exact GP
def scaled(x, length_scale):
    """x / ls in fp64 from the fp32 inputs (sklearn's RBF divides by the length scale before scipy's distance)."""
    return np.asarray(x, dtype=np.float32).astype(np.float64) / float(length_scale)


def rbf_matrix(xa, xb, length_scale):
    a, b = scaled(xa, length_scale), scaled(xb, length_scale)
    d2 = ((a[:, None, :] - b[None, :, :]) ** 2).sum(-1)
    return np.exp(-0.5 * d2)


def exact_gp_ref(x, y, length_scale, alpha=ALPHA_GP):
    """mean, var [T] (index 0 NaN), status (0 or the first prefix whose factor fails) and per prefix the quantities of
    exact_gp_bound: GaussianProcessRegressor(RBF(ls), alpha).fit(x[:t], y[:t]).predict(x[t]), var clipped at 0."""
    x = np.asarray(x, dtype=np.float32)
    y = np.asarray(y, dtype=np.float64)
    T = x.shape[0]
    K = rbf_matrix(x, x, length_scale)
    mean, var = np.full(T, np.nan), np.full(T, np.nan)
    info = [None]
    for t in range(1, T):
        A = K[:t, :t] + alpha * np.eye(t)
        try:
            Lc = np.linalg.cholesky(A)
        except np.linalg.LinAlgError:
            return mean, var, t, info
        ks = K[:t, t]
        v = np.linalg.solve(Lc, ks)
        zy = np.linalg.solve(Lc, y[:t])
        mean[t] = v @ zy
        var[t] = max(1.0 - v @ v, 0.0)
        a = np.linalg.solve(Lc.T, v)
        ay = np.linalg.solve(Lc.T, zy)
        info.append(dict(t=t, a=np.linalg.norm(a), ay=np.linalg.norm(ay), ks=np.linalg.norm(ks), normA=np.linalg.norm(A, 2)))
    return mean, var, 0, info


def exact_gp_bound(info):
    """Per-element bounds (mean, var) on |device - ref| from a backward error gamma = 8 t eps |A| of both Cholesky
    solves: |dmean| <= gamma |A^-1 k*| |A^-1 y| + eps-level kernel errors, |dvar| <= gamma |A^-1 k*|^2 + the same."""
    bm, bv = np.full(len(info), np.nan), np.full(len(info), np.nan)
    for t, d in enumerate(info):
        if d is None:
            continue
        g = 8.0 * d["t"] * EPS * d["normA"]
        k_err = 8.0 * EPS * d["ks"]
        bm[t] = 2 * (g * d["a"] * d["ay"] + k_err * d["ay"] + EPS)
        bv[t] = 2 * (g * d["a"] ** 2 + 2 * k_err * d["a"] + EPS)
    return bm, bv


def gp_losses(mean, var, y, use_mse=False, var_eps=1e-6):
    """Per-t loss of priors/gp.py evaluate: GaussianNLLLoss(full=True) with var clamped at eps, or the squared error."""
    y = np.asarray(y, dtype=np.float64)
    if use_mse:
        return (mean - y) ** 2
    v = np.maximum(var, var_eps)
    return 0.5 * (np.log(v) + (y - mean) ** 2 / v) + 0.5 * LOG_2PI


def gp_loss_bound(mean, var, y, bm, bv, use_mse=False, var_eps=1e-6):
    """Bound on the loss difference implied by |dmean| <= bm and |dvar| <= bv (the clamp only shrinks it)."""
    e = np.abs(np.asarray(y, dtype=np.float64) - mean)
    if use_mse:
        return bm * (2 * e + bm)
    v = np.maximum(var, var_eps)
    return 0.5 * bv / v + (e * bm + 0.5 * bm ** 2) / v + 0.5 * (e + bm) ** 2 * bv / (v * v) * 2


def pivoted_cholesky_ref(x, length_scale):
    """(factor [T, T] = P L in the rows' own order, perm [T], rank) of K = RBF(x, x): diagonal pivoting, ties to the
    smallest row, stopping at the first step whose largest remaining diagonal is at or below T eps."""
    x = np.asarray(x, dtype=np.float32)
    T = x.shape[0]
    K = rbf_matrix(x, x, length_scale)
    G = np.zeros((T, T))
    d = np.ones(T)
    chosen = np.zeros(T, dtype=bool)
    perm = []
    for k in range(T):
        cand = np.where(chosen, -1.0, d)
        p = int(np.argmax(cand))
        if not cand[p] > T * EPS:
            break
        piv = np.sqrt(cand[p])
        col = (K[:, p] - G[:, :k] @ G[p, :k]) / piv
        col[chosen] = 0.0
        col[p] = piv
        G[:, k] = col
        d = d - col ** 2
        chosen[p] = True
        perm.append(p)
    rank = len(perm)
    perm += [i for i in range(T) if not chosen[i]]
    return G, np.array(perm), rank
