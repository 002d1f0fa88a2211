"""`tabular` (reference tabular.py): the tabular evaluation of the PFN checkpoints and of the KNN baseline.

The module keeps the reference's public names, signatures, prints and result-dict keys, so TabularEvalSimple.ipynb runs
against it (`install_dropin()` registers it as `tabular`).  Two paths run on the device:

* the PFN (this package's `TransformerModel`): `evaluate_position` scores all Q = bptt - eval_position test rows of all
  S samples in ONE forward pass, as Q * S contexts of p + 1 rows (the reference runs one pass per test row).  Context
  (q, s) is the p train rows of sample s plus its test row p + q, standardised with the mean and unbiased std (+ 1e-6)
  of those p + 1 rows and divided by `rescale_features` (reference :289-296).  The statistics are fp64 (from the train
  prefix's, once per sample) and the standardised values are rounded to fp32 once: a column that is constant in a
  context gives exactly 0, where the reference's fp32 mean can be off by an ulp, amplified by 1 / 1e-6;
* the KNN baseline: `batch_pred` recognises `knn_metric` and runs the grid-search CV and refit of all S samples in one
  launch of csrc/knn_cv.cu.

The metric is ROC AUC in the Mann-Whitney form, computed here without sklearn.  Any other `nn.Module` keeps the
reference's per-position loop, and any other callable runs per sample through `batch_pred` (host glue).  The GP-classifier,
logistic-regression, Bayesian-NN, CatBoost and XGBoost baselines are not provided (NotImplementedError), nor plotting,
OpenML loading (`datasets`) or the command line.
"""
import os
import random
import time

import numpy as np
import torch
from torch import nn

from . import _lib as L
from . import encoders, priors
from .priors.utils import gamma_sampler_f, trunc_norm_sampler_f
from .train import Losses, train
from .transformer import TransformerModel

CV = 5
param_grid = {}
RESULTS_DIR = '/home/anon/prior-fitting/results/tabular'   # where `evaluate` caches per-dataset results (reference :168)
MAX_FORWARD_TOKENS = 1 << 20     # tokens (T * B) of one PFN forward; larger batches of contexts are split


def roc_auc(y_true, y_score):
    """ROC AUC of every group along the last axis: y_true, y_score [..., n] -> [...] fp64 (a numpy float for 1-d inputs).
    Mann-Whitney form: the share of (positive, negative) pairs whose positive scores higher, ties counting one half.
    Raises ValueError when a group holds one class only, or labels other than 0 / 1."""
    y = torch.as_tensor(np.asarray(y_true), dtype=torch.float64)
    p = torch.as_tensor(np.asarray(y_score), dtype=torch.float64)
    if not bool(((y == 0) | (y == 1)).all()):
        raise ValueError("roc_auc: labels must be 0 or 1")
    pos, neg = y == 1, y == 0
    n_pos, n_neg = pos.sum(-1), neg.sum(-1)
    if bool(((n_pos == 0) | (n_neg == 0)).any()):
        raise ValueError("Only one class present in y_true. ROC AUC score is not defined in that case.")
    d = p.unsqueeze(-1) - p.unsqueeze(-2)                   # [..., i, j] = score_i - score_j
    pair = (pos.unsqueeze(-1) & neg.unsqueeze(-2)).long()
    twice = ((2 * (d > 0).long() + (d == 0).long()) * pair).sum((-2, -1))
    return (twice.double() / (2.0 * n_pos.double() * n_neg.double())).numpy()[()]


metric_used = roc_auc


def get_uniform_single_eval_pos_sampler(max_len):
    """Every evaluation position in [0, max_len) with the same weight (reference :39-44)."""
    return lambda: random.choices(range(max_len))[0]


def _first(sampler_dict):
    return next(iter(sampler_dict.values()))


def get_mlp_prior_hyperparameters(config):
    """The 17-tuple `priors.mlp` takes (reference :47-70); the causal entries are None unless 'prior_is_causal'."""
    causal = config['prior_is_causal']
    if_causal = lambda read: read() if causal else None
    return (_first(config['prior_nlayers_sampler']),
            _first(config['prior_emsize_sampler']),
            config['prior_activations'],
            gamma_sampler_f(config['prior_sigma_gamma_k'], config['prior_sigma_gamma_theta']),
            gamma_sampler_f(config['prior_noise_std_gamma_k'], config['prior_noise_std_gamma_theta']),
            _first(config['prior_dropout_sampler']),
            True,
            _first(config['prior_num_features_used_sampler']),
            if_causal(lambda: _first(config['prior_causes_sampler'])),
            causal,
            if_causal(lambda: config['prior_pre_sample_causes']),
            if_causal(lambda: config['prior_pre_sample_weights']),
            if_causal(lambda: config['prior_y_is_effect']),
            config['prior_order_y'],
            config['prior_normalize_by_used_features'],
            if_causal(lambda: _first(config['prior_categorical_feats'])),
            0.0)


def get_gp_mix_prior_hyperparameters(config):
    """The hyperparameter dict of `priors.fast_gp_mix` (reference :73-80), quirks included: 'categorical_data' reads
    prior_y_minmax_norm and 'y_minmax_norm' reads prior_lengthscale_concentration."""
    return {'lengthscale_concentration': config['prior_lengthscale_concentration'],
            'nu': config['prior_nu'],
            'outputscale_concentration': config['prior_outputscale_concentration'],
            'categorical_data': config['prior_y_minmax_norm'],
            'y_minmax_norm': config['prior_lengthscale_concentration'],
            'noise_concentration': config['prior_noise_concentration'],
            'noise_rate': config['prior_noise_rate']}


def _gp_tuple(config, outputscale_sampler, lengthscale_sampler):
    return (config['prior_noise'], outputscale_sampler, lengthscale_sampler, True,
            _first(config['prior_num_features_used_sampler']), config['prior_normalize_by_used_features'],
            config['prior_order_y'])


def get_gp_prior_hyperparameters(config):
    """The 7-tuple of `priors.fast_gp` with fixed outputscale and lengthscale (reference :83-92)."""
    return _gp_tuple(config, lambda: config['prior_outputscale'], lambda: config['prior_lengthscale'])


def get_meta_gp_prior_hyperparameters(config):
    """The 7-tuple of `priors.fast_gp` with truncated-normal outputscale and lengthscale samplers (reference :95-105)."""
    ls = trunc_norm_sampler_f(config['prior_lengthscale_mean'], config['prior_lengthscale_mean'] * config['prior_lengthscale_std_f'])
    os_ = trunc_norm_sampler_f(config['prior_outputscale_mean'], config['prior_outputscale_mean'] * config['prior_outputscale_std_f'])
    return _gp_tuple(config, os_, ls)


def get_model(config, device, eval_positions, should_train=True, verbose=False):
    """`train()` under the BCE loss on the prior `config['prior_type']` names ('mlp', 'gp', 'custom_gp_mix', 'gp_mix'),
    zero epochs when not `should_train` (reference :109-155).  Returns what `train` returns: (loss, positional losses,
    model).  With zero epochs the prior is never sampled, so a config whose samplers are placeholders still builds."""
    extra_kwargs = {}
    prior_type = config['prior_type']
    if prior_type == 'mlp':
        hyperparameters, prior = get_mlp_prior_hyperparameters(config), priors.mlp.DataLoader
        extra_kwargs['batch_size_per_gp_sample'] = 8
    elif prior_type == 'gp':
        hyperparameters, prior = get_gp_prior_hyperparameters(config), priors.fast_gp.DataLoader
    elif prior_type == 'custom_gp_mix':
        hyperparameters, prior = get_meta_gp_prior_hyperparameters(config), priors.fast_gp.DataLoader
    elif prior_type == 'gp_mix':
        hyperparameters, prior = get_gp_mix_prior_hyperparameters(config), priors.fast_gp_mix.DataLoader
    else:
        raise Exception(f"unknown prior_type {prior_type!r}")
    epochs = config['epochs'] if should_train else 0
    return train(prior, Losses.bce, encoders.Linear, emsize=config['emsize'], nhead=config['nhead'],
                 y_encoder_generator=encoders.Linear, pos_encoder_generator=None, batch_size=config['batch_size'],
                 nlayers=config['nlayers'], nhid=config['emsize'] * config['nhid_factor'], epochs=epochs,
                 warmup_epochs=epochs // 4, bptt=config['bptt'], gpu_device=device, dropout=config['dropout'],
                 steps_per_epoch=100, single_eval_pos_gen=get_uniform_single_eval_pos_sampler(max(eval_positions) + 1),
                 extra_prior_kwargs_dict={'num_features': config['num_features'], 'fuse_x_y': False,
                                          'hyperparameters': hyperparameters, **extra_kwargs},
                 lr=config['lr'], verbose=verbose)


def get_default_spec(test_datasets, valid_datasets):
    """(bptt, eval_positions, max_features, max_samples) of the paper's evaluation (reference :628-634)."""
    max_features = max(X.shape[1] for (_, X, _, _) in list(test_datasets) + list(valid_datasets))
    return 100, [30], max_features, 20


# ---- evaluation (reference :160-323) ---------------------------------------------------------------------------------
def evaluate(datasets, model, method, bptt, eval_position_range, device, max_features=0, plot=False, extend_features=False,
             save=True, rescale_features=False, overwrite=False, max_samples=40, path_interfix=''):
    """Scores `model` (a PFN, or a per-sample metric function such as `knn_metric`) on every [name, X, y, categorical_feats]
    of `datasets` at every eval position (reference :160-213).  Per dataset the result holds
    '{name}_mean_metric_at_{pos}' (the AUC over all samples' outputs) and '{name}_time', with `save` also
    '{name}_per_ds_metric_at_{pos}', '_outputs_at_' and '_ys_at_', and the dataset's dict is cached in
    RESULTS_DIR/{path_interfix}/results_{method}_{name}.npy (reused unless `overwrite`).  Then 'mean_metric_at_{pos}'
    over datasets and 'mean_metric'.  The PFN and the KNN baseline run on a CUDA device: `device='cpu'` selects the
    current one; results are numpy arrays and tensors on `device`."""
    if plot:
        raise NotImplementedError("plot=True: plotting (matplotlib) is not provided")
    result = {'metric': 'auc'}
    for [name, X, y, categorical_feats] in datasets:
        result_ds = {}
        path = f'{RESULTS_DIR}/{path_interfix}/results_{method}_{name}.npy'
        if os.path.isfile(path) and not overwrite:
            with open(path, 'rb') as f:
                result_ds = np.load(f, allow_pickle=True).tolist()
            if 'time' in result_ds:
                result_ds[name + '_time'] = result_ds.pop('time')
            result.update(result_ds)
            mean_metric = float(result[name + '_mean_metric_at_' + str(eval_position_range[-1])])
            print(f'Loaded saved result for {name} (mean metric {mean_metric})')
            continue

        print('Evaluating ' + str(name))
        rescale_features_factor = X.shape[1] / max_features if rescale_features and extend_features else 1.0
        if extend_features:
            X = torch.cat([X, torch.zeros((X.shape[0], max_features - X.shape[1]))], -1)
        start_time = time.time()
        ds_result = evaluate_dataset(X.to(device), y.to(device), categorical_feats, model, bptt, eval_position_range,
                                     rescale_features=rescale_features_factor, max_samples=max_samples)
        elapsed = time.time() - start_time
        for pos, (metric, outputs, ys) in zip(eval_position_range, ds_result):
            if save:
                result_ds[f'{name}_per_ds_metric_at_{pos}'] = metric
                result_ds[f'{name}_outputs_at_{pos}'] = outputs
                result_ds[f'{name}_ys_at_{pos}'] = ys
            result_ds[f'{name}_mean_metric_at_{pos}'] = metric_used(ys.detach().cpu().flatten(), outputs.flatten())
            result_ds[name + '_time'] = elapsed
        if save:
            with open(path, 'wb') as f:
                np.save(f, result_ds)
        result.update(result_ds)

    for pos in eval_position_range:
        result[f'mean_metric_at_{pos}'] = np.array([result[f'{d[0]}_mean_metric_at_{pos}'] for d in datasets]).mean()
    result['mean_metric'] = np.array([result[f'mean_metric_at_{pos}'] for pos in eval_position_range]).mean()
    return result


def evaluate_dataset(X, y, categorical_feats, model, bptt, eval_position_range, plot=False, rescale_features=1.0,
                     max_samples=40):
    """`evaluate_position` at every eval position (reference :216-228): a list of (metric, outputs, ys)."""
    if plot:
        raise NotImplementedError("plot=True: plotting (matplotlib) is not provided")
    result = []
    for eval_position in eval_position_range:
        result.append(evaluate_position(X, y, categorical_feats, model, bptt, eval_position,
                                        rescale_features=rescale_features, max_samples=max_samples))
        print('\t Eval position ' + str(eval_position) + ' done..')
    return result


def eval_windows(X, y, bptt, max_samples):
    """The windows X[i:i+bptt] for i < len(X) - bptt stacked on dim 1 ([bptt, N, F], [bptt, N]), then at most
    `max_samples` of them chosen by torch.randperm on a CPU generator seeded 13 (reference :238-277: the same permutation
    as manual_seed(13) under fork_rng, without touching the global generators)."""
    num_evals = len(X) - bptt
    if num_evals <= 0:
        raise ValueError(f"a dataset of {len(X)} rows has no window of bptt + 1 = {bptt + 1} rows")
    eval_xs = torch.stack([X[i:i + bptt] for i in range(num_evals)], 1)
    eval_ys = torch.stack([y[i:i + bptt] for i in range(num_evals)], 1)
    sel = torch.randperm(eval_xs.shape[1], generator=torch.Generator().manual_seed(13))[:max_samples]
    return eval_xs[:, sel.to(eval_xs.device), :], eval_ys[:, sel.to(eval_ys.device)]


def evaluate_position(X, y, categorical_feats, model, bptt, eval_position, rescale_features=1.0, max_samples=40):
    """(metric per sample [S], outputs [Q, S], ys [Q, S]) at one eval position (reference :231-306): the first
    `eval_position` rows of each window train, the Q = bptt - eval_position others are scored."""
    eval_xs, eval_ys = eval_windows(X, y, bptt, max_samples)
    p = eval_position
    if isinstance(model, TransformerModel):
        outputs = _pfn_outputs(model, eval_xs, eval_ys, p, rescale_features)
    elif isinstance(model, nn.Module):
        outputs = _module_outputs(model, eval_xs, eval_ys, p, rescale_features)
    else:
        metric, outputs = batch_pred(model, eval_xs, eval_ys, categorical_feats, start=p)
        return metric, outputs, eval_ys[p:]
    metric_per_t = metric_used(eval_ys[p:].detach().cpu().T, outputs.T)
    return metric_per_t, outputs, eval_ys[p:]


def _module_outputs(model, eval_xs, eval_ys, p, rescale_features):
    """The reference's loop (:285-300) for a module other than this package's TransformerModel: one pass per test row."""
    model.eval()
    outputs = np.zeros((eval_xs.shape[0] - p, eval_xs.shape[1]))
    for i, pos in enumerate(range(p, eval_xs.shape[0])):
        eval_x = torch.cat([eval_xs[:p], eval_xs[pos].unsqueeze(0)])
        eval_x = (eval_x - eval_x.mean(0)) / (eval_x.std(0) + .000001) / rescale_features
        output = torch.sigmoid(model((eval_x, eval_ys[:p].float()), single_eval_pos=p)).squeeze(-1)
        outputs[i, :] = output.detach().cpu().numpy()
    return outputs


_PFN = "the tabular PFN evaluation runs this package's TransformerModel on sm_90a kernels"


def pfn_contexts(eval_xs, eval_ys, p, rescale_features=1.0):
    """The Q * S contexts of one eval position: x [p + 1, Q * S, F] fp32, y [p + 1, Q * S] fp32 (row p is 0 and unused).
    Column b = q * S + s is sample s's p train rows plus its test row p + q, standardised with the mean and unbiased
    std (+ 1e-6) of those p + 1 rows (fp64, from the train prefix's statistics) and divided by rescale_features."""
    T, S, F = eval_xs.shape
    Q = T - p
    x = eval_xs.double()
    prefix = x[:p]
    m0 = prefix.mean(0)                                       # [S, F]
    c0 = ((prefix - m0) ** 2).sum(0)                          # [S, F]
    test = x[p:]                                              # [Q, S, F]
    delta = test - m0
    mean = m0 + delta / (p + 1)                               # [Q, S, F]: statistics of train rows + test row q
    var = (c0 + delta * (test - mean)) / p
    std = var.clamp_min(0).sqrt() + 1e-6
    ctx = torch.cat([prefix.unsqueeze(1).expand(p, Q, S, F), test.unsqueeze(0)], 0)   # [p + 1, Q, S, F]
    xs = ((ctx - mean) / std / rescale_features).float().reshape(p + 1, Q * S, F)
    ys = torch.zeros(p + 1, Q * S, dtype=torch.float32, device=eval_ys.device)
    ys[:p] = eval_ys[:p].float().unsqueeze(1).expand(p, Q, S).reshape(p, Q * S)
    return xs, ys


@torch.no_grad()
def _pfn_outputs(model, eval_xs, eval_ys, p, rescale_features):
    """sigmoid of the PFN's output for every test row of every sample, all contexts in one forward pass (split into
    chunks of whole contexts only past MAX_FORWARD_TOKENS tokens): numpy fp64 [Q, S]."""
    dev = L.compute_device(eval_xs.device, _PFN)
    home = next(model.parameters()).device
    model.eval()
    model.to(dev)
    try:
        T, S, _ = eval_xs.shape
        xs, ys = pfn_contexts(eval_xs.to(dev), eval_ys.to(dev), p, rescale_features)
        per = max(1, MAX_FORWARD_TOKENS // (p + 1))
        logits = torch.cat([model((xs[:, b:b + per].contiguous(), ys[:, b:b + per].contiguous()), single_eval_pos=p)
                            for b in range(0, xs.shape[1], per)], 1)
        out = torch.sigmoid(logits.float()).squeeze(-1).squeeze(0).reshape(T - p, S)
        return out.double().cpu().numpy()
    finally:
        model.to(home)


def batch_pred(metric_function, eval_xs, eval_ys, categorical_feats, start=2):
    """Per sample: x standardised with its train prefix's mean and unbiased std (+ 1e-6), then
    metric_function(train_x, train_y, test_x, test_y, categorical_feats) -> (metric, outputs) (reference :309-323).
    Returns (metrics [S], outputs [Q, S]) as numpy arrays.  `knn_metric` runs all samples in one device launch."""
    if metric_function is knn_metric:
        proba, _, _ = knn_cv(standardize_by_prefix(eval_xs, start), eval_ys[:start])
        outputs = proba.cpu().numpy()
        return metric_used(eval_ys[start:].detach().cpu().T, outputs.T), outputs
    metrics, outputs = [], []
    for eval_x, eval_y in zip(eval_xs.transpose(0, 1), eval_ys.transpose(0, 1)):
        mean = eval_x[:start].mean(0)
        std = eval_x[:start].std(0) + .000001
        eval_x = (eval_x - mean) / std
        metric, output = metric_function(eval_x[:start], eval_y[:start], eval_x[start:], eval_y[start:], categorical_feats)
        metrics.append(metric)
        outputs.append(output)
    return np.array(metrics), np.array(outputs).T


def standardize_by_prefix(eval_xs, start):
    """x [T, S, F] standardised with the mean and unbiased std (+ 1e-6) of its first `start` rows, statistics in fp64,
    the result rounded to fp32."""
    x = eval_xs.double()
    prefix = x[:start]
    return ((x - prefix.mean(0)) / (prefix.std(0) + 1e-6)).float()


# ---- KNN (reference :349-369) ------------------------------------------------------------------------------------------
param_grid['knn'] = {'n_neighbors (max number of samples)': np.arange(1, 6)}
_KNN = "the KNN baseline runs on the sm_90a kernel of csrc/knn_cv.cu"
_KNN_ERRORS = {
    L.KNN_BAD_LABEL: "labels must be 0 or 1",
    L.KNN_FEW_MEMBERS: "n_splits={ns} cannot be greater than the number of members in each class",
    L.KNN_ONE_CLASS: "the training labels hold one class only, so there is no class-1 probability",
}


@torch.no_grad()
def knn_cv(x, y):
    """The KNN grid search of `knn_metric` for S problems in one launch: x [n + m, S, F] (already standardised),
    y [n, S] (0 / 1).  Returns (proba [m, S] fp64, k_best [S] int32, cv_mean [S, K] fp64), K = min(5, n - 2), on the
    CUDA device that ran them.  Raises ValueError for a problem sklearn's GridSearchCV rejects (or whose refit has one
    class only, where the reference fails in `predict_proba(...)[:, 1]`)."""
    rows, S, F = x.shape
    n = y.shape[0]
    m = rows - n
    if n // 2 < 2:
        raise ValueError(f"knn_metric: n={n} training rows give n // 2 = {n // 2} < 2 cross-validation folds")
    if n > L.KNN_MAX_N or F > L.KNN_MAX_F:
        raise ValueError(f"knn_metric: n={n} rows, F={F} features: the kernel takes at most {L.KNN_MAX_N} rows and "
                         f"{L.KNN_MAX_F} features")
    if m < 1:
        raise ValueError("knn_metric: no test rows")
    dev = L.compute_device(x.device, _KNN)
    K = min(L.KNN_MAX_K, n - 2)
    with L.on_device(dev):
        proba = torch.empty(m, S, dtype=torch.float64, device=dev)
        k_best = torch.empty(S, dtype=torch.int32, device=dev)
        cv_mean = torch.empty(S, K, dtype=torch.float64, device=dev)
        status = torch.empty(S, dtype=torch.int32, device=dev)
        L.knn_cv(x.to(dev, torch.float32).contiguous(), y.to(dev, torch.float32).contiguous(), proba, k_best, cv_mean, status)
        status = status.cpu()
    bad = torch.nonzero(status).flatten()
    if len(bad):
        s = int(bad[0])
        raise ValueError(f"knn_metric: sample {s}: " + _KNN_ERRORS[int(status[s])].format(ns=min(CV, n // 2)))
    return proba, k_best, cv_mean


def knn_metric(x, y, test_x, test_y, cat_features):
    """GridSearchCV over n_neighbors 1 .. min(5, n - 2) with min(5, n // 2) stratified folds, then the refit's class-1
    probabilities of test_x (reference :351-369), as a one-problem launch.  -> (AUC, proba [m] numpy)."""
    xs = torch.cat([x, test_x], 0).unsqueeze(1)
    proba, _, _ = knn_cv(xs, y.unsqueeze(1))
    pred = proba[:, 0].cpu().numpy()
    return metric_used(test_y.cpu().numpy(), pred), pred


# ---- baselines this package does not provide ------------------------------------------------------------------------
def _not_provided(name, what):
    def fn(x, y, test_x, test_y, cat_features):
        raise NotImplementedError(f"{name}: the {what} baseline is not provided by this package (knn_metric is)")
    fn.__name__ = fn.__qualname__ = name
    return fn


logistic_metric = _not_provided('logistic_metric', 'sklearn LogisticRegression grid-search')
gp_metric = _not_provided('gp_metric', 'sklearn GaussianProcessClassifier grid-search')
bayes_net_metric = _not_provided('bayes_net_metric', 'pyro SVI Bayesian-NN')
catboost_metric = _not_provided('catboost_metric', 'CatBoost')
xgb_metric = _not_provided('xgb_metric', 'XGBoost')


class BayesianModel:
    """The reference's pyro Bayesian NN of the tabular baselines (:373-411): not provided."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError("tabular.BayesianModel (pyro) is not provided by this package")


class BayesianNNClassifier:
    """The reference's sklearn wrapper of the pyro Bayesian NN (:414-462): not provided."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError("tabular.BayesianNNClassifier (pyro SVI) is not provided by this package")
