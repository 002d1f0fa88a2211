"""fp64 restatement of the tabular evaluation (reference tabular.py:160-369) for the tests of
transformerscandobayesianinference_b200.tabular: the eval windows and their seed-13 selection, the per-context
standardisation of the PFN path, sklearn's StratifiedKFold (_make_test_folds, no shuffling) and the KNN grid search
with its refit, and the Mann-Whitney ROC AUC.  numpy / torch on the CPU only; the model forward is
pfn_oracle.transformer_forward_ref.  TEST INFRASTRUCTURE ONLY.
"""
import numpy as np
import torch

from oracle import pfn_oracle as O


def windows(X, y, bptt, max_samples):
    """[bptt, S, F], [bptt, S]: the windows X[i:i+bptt], i < len(X) - bptt, of the torch.randperm (seed 13) selection."""
    n = len(X) - bptt
    xs = torch.stack([torch.as_tensor(X[i:i + bptt]) for i in range(n)], 1)
    ys = torch.stack([torch.as_tensor(y[i:i + bptt]) for i in range(n)], 1)
    sel = torch.randperm(n, generator=torch.Generator().manual_seed(13))[:max_samples]
    return xs[:, sel], ys[:, sel]


def pfn_contexts_ref(eval_xs, eval_ys, p, rescale=1.0):
    """fp64 [p + 1, Q * S, F] contexts (column q * S + s: train rows of sample s plus its test row p + q), each standardised
    by the two-pass mean and unbiased std (+ 1e-6) of its own p + 1 rows, then / rescale; y [p, Q * S]."""
    x = torch.as_tensor(eval_xs).double()
    T, S, F = x.shape
    Q = T - p
    ctx = torch.cat([x[:p].unsqueeze(1).expand(p, Q, S, F), x[p:].unsqueeze(0)], 0)
    mean = ctx.mean(0)
    std = ((ctx - mean) ** 2).sum(0).div(p).sqrt() + 1e-6
    xs = ((ctx - mean) / std / rescale).reshape(p + 1, Q * S, F)
    ys = torch.as_tensor(eval_ys[:p]).double().unsqueeze(1).expand(p, Q, S).reshape(p, Q * S)
    return xs, ys


def pfn_outputs_ref(P, nhead, eval_xs, eval_ys, p, rescale=1.0):
    """sigmoid of the fp64 model forward on every context: [Q, S] fp64."""
    T, S = eval_xs.shape[:2]
    xs, ys = pfn_contexts_ref(eval_xs, eval_ys, p, rescale)
    ys = torch.cat([ys, torch.zeros(1, ys.shape[1], dtype=ys.dtype)], 0)
    logits = O.transformer_forward_ref(P, xs, ys, p, nhead)
    return torch.sigmoid(logits[0, :, 0]).reshape(T - p, S).numpy()


def seeded_state_dict(model, seed):
    """Weights for a TransformerModel (the reference's or this package's: the keys are the same) drawn from one generator
    seeded `seed`, key by key in sorted order, so the goldens need not store them: LayerNorm weights 1 + 0.1 N(0, 1),
    other vectors 0.1 N(0, 1), matrices 0.5 N(0, 1) / sqrt(fan_in)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k in sorted(model.state_dict()):
        t = model.state_dict()[k]
        z = torch.randn(t.shape, generator=g, dtype=torch.float32)
        if t.dim() == 2:
            out[k] = 0.5 * z / t.shape[1] ** 0.5
        else:
            out[k] = 1.0 + 0.1 * z if ("norm" in k and k.endswith("weight")) else 0.1 * z
    return out


def checksum(sd):
    """(sum, sum of |.|) in fp64 of every tensor: proof that two state dicts were built alike."""
    return {k: (float(v.double().sum()), float(v.double().abs().sum())) for k, v in sd.items()}


def auc(y, s):
    """Mann-Whitney ROC AUC of one group (ties count one half)."""
    y, s = np.asarray(y, dtype=np.float64), np.asarray(s, dtype=np.float64)
    pos, neg = s[y == 1], s[y == 0]
    if len(pos) == 0 or len(neg) == 0:
        raise ValueError("one class only")
    d = pos[:, None] - neg[None, :]
    return ((d > 0).sum() + 0.5 * (d == 0).sum()) / (len(pos) * len(neg))


def auc_interval(y, s, bound):
    """(lo, hi): the AUC when the pairs whose scores are within `bound` of each other all count against / for."""
    y, s = np.asarray(y, dtype=np.float64), np.asarray(s, dtype=np.float64)
    d = s[y == 1][:, None] - s[y == 0][None, :]
    return (d > bound).sum() / d.size, (d >= -bound).sum() / d.size


def stratified_folds(y, n_splits):
    """Test-fold index of every row, as sklearn's StratifiedKFold(n_splits)._make_test_folds without shuffling."""
    y = np.asarray(y)
    _, first, inv = np.unique(y, return_index=True, return_inverse=True)
    enc = np.argsort(np.argsort(first))[inv]                  # classes by order of first appearance
    n_classes = len(first)
    counts = np.bincount(enc)
    if np.all(n_splits > counts):
        raise ValueError(f"n_splits={n_splits} cannot be greater than the number of members in each class.")
    order = np.sort(enc)
    alloc = np.asarray([np.bincount(order[i::n_splits], minlength=n_classes) for i in range(n_splits)])
    folds = np.empty(len(y), dtype=int)
    for k in range(n_classes):
        folds[enc == k] = np.arange(n_splits).repeat(alloc[:, k])
    return folds


def sq_dists(a, b):
    """Squared Euclidean distances [len(a), len(b)] in fp64, summed feature by feature from direct differences."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    d = np.zeros((len(a), len(b)))
    for f in range(a.shape[1]):
        t = a[:, f][:, None] - b[:, f][None, :]
        d = d + t * t
    return d


def _neighbour_ones(d, y_train, k):
    """Class-1 count among the k nearest (by (distance, index)) of every row of d [q, n]."""
    order = np.argsort(d, axis=1, kind='stable')[:, :k]
    return np.asarray(y_train)[order].sum(1)


def knn_grid_search(x, y, test_x):
    """GridSearchCV(KNeighborsClassifier(), n_neighbors 1 .. min(5, n - 2), cv=min(5, n // 2)) + predict_proba[:, 1],
    restated: returns (proba [m], k, cv_mean [K], gap [m]) where gap is the relative gap between the k-th and (k+1)-th
    squared distances of each test row (inf when there is no (k+1)-th row)."""
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y).astype(int)
    n = len(y)
    ns = min(5, n // 2)
    if ns < 2:
        raise ValueError("n // 2 < 2")
    if not np.isin(y, (0, 1)).all():
        raise ValueError("labels outside {0, 1}")
    folds = stratified_folds(y, ns)
    if len(np.unique(y)) == 1:
        raise ValueError("one class only")
    ks = np.arange(1, min(6, n - 1))
    D = sq_dists(x, x)
    scores = np.full((len(ks), ns), np.nan)
    for f in range(ns):
        te, tr = folds == f, folds != f
        d = D[np.ix_(te, tr)]
        for i, k in enumerate(ks):
            if k > tr.sum():
                continue
            ones = _neighbour_ones(d, y[tr], k)
            pred = (2 * ones > k).astype(int)
            scores[i, f] = (pred == y[te]).sum() / te.sum()
    means = scores.mean(1)
    valid = ~np.isnan(means)
    best = int(np.flatnonzero(valid & (means == np.nanmax(means)))[0]) if valid.any() else 0
    k = int(ks[best])
    dt = sq_dists(test_x, x)
    proba = _neighbour_ones(dt, y, k) / k
    srt = np.sort(dt, 1)
    gap = np.full(len(dt), np.inf) if n <= k else (srt[:, k] - srt[:, k - 1]) / np.maximum(srt[:, k], 1e-300)
    return proba, k, means, gap


def standardize_by_prefix(eval_xs, start):
    """x [T, S, F] standardised by the fp64 mean and unbiased std (+ 1e-6) of the first `start` rows, rounded to fp32."""
    x = torch.as_tensor(eval_xs).double()
    pre = x[:start]
    return ((x - pre.mean(0)) / (pre.std(0) + 1e-6)).float()


def knn_position_ref(eval_xs, eval_ys, p):
    """knn_grid_search on every sample of one eval position (inputs standardised as the device path does):
    proba [Q, S], k [S], cv_mean [S, K], gap [Q, S]."""
    xs = standardize_by_prefix(eval_xs, p).numpy()
    ys = np.asarray(eval_ys)
    res = [knn_grid_search(xs[:p, s], ys[:p, s], xs[p:, s]) for s in range(xs.shape[1])]
    return (np.stack([r[0] for r in res], 1), np.array([r[1] for r in res]), np.stack([r[2] for r in res]),
            np.stack([r[3] for r in res], 1))
