"""The tabular evaluation (`tabular`) on the host: the fp64 oracle's KNN grid search and AUC against sklearn, the harness
(windows, seed-13 selection, result keys and types, feature extension, the .npy cache) against the reference's goldens
(tests/golden/tabular.pt, written by oracle/make_tabular_golden.py), the setup helpers and the baselines not provided."""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import transformerscandobayesianinference_b200 as pfn  # noqa: E402
from transformerscandobayesianinference_b200 import tabular  # noqa: E402
from oracle import error_budget as EB, tabular_oracle as T  # noqa: E402

GOLDEN = torch.load(os.path.join(ROOT, "tests", "golden", "tabular.pt"), weights_only=False)


def _random_problem(rng, trial):
    n = int(rng.integers(6, 100))
    y = (rng.random(n) < rng.uniform(0.1, 0.9)).astype(int)
    if y.min() == y.max():
        y[rng.integers(n)] ^= 1
    if trial % 2:
        y = 1 - y
    x = rng.normal(size=(n + 5, int(rng.integers(1, 8)))).astype(np.float32)
    return n, x, y


def test_oracle_knn_matches_sklearn_grid_search():
    sk = pytest.importorskip("sklearn")  # noqa: F841
    from sklearn.model_selection import GridSearchCV
    from sklearn.neighbors import KNeighborsClassifier
    warnings.filterwarnings("ignore")
    rng = np.random.default_rng(0)
    checked = 0
    for trial in range(520):
        n, x, y = _random_problem(rng, trial)
        try:
            clf = GridSearchCV(KNeighborsClassifier(), {'n_neighbors': np.arange(1, min(6, n - 1))},
                               cv=min(5, n // 2)).fit(x[:n], y)
        except ValueError:
            with pytest.raises(ValueError):
                T.knn_grid_search(x[:n], y, x[n:])
            continue
        proba, k, means, _ = T.knn_grid_search(x[:n], y, x[n:])
        assert k == clf.best_params_['n_neighbors'], trial
        assert np.array_equal(means, clf.cv_results_['mean_test_score'], equal_nan=True), trial
        np.testing.assert_array_equal(proba, clf.predict_proba(x[n:])[:, 1])
        checked += 1
    assert checked >= 500


def test_oracle_knn_matches_golden_choices():
    """On the fixture's datasets the oracle (fp64 standardisation) chooses sklearn's k with sklearn's CV means, except
    where the two standardisations move a sample across a near-tie."""
    agree = total = 0
    for (name, p), rec in GOLDEN["knn"].items():
        X, y = next((d[1], d[2]) for d in GOLDEN["datasets"] if d[0] == name)
        eval_xs, eval_ys = T.windows(X, y, GOLDEN["bptt"], GOLDEN["max_samples"])
        _, k, cv_mean, _ = T.knn_position_ref(eval_xs, eval_ys, p)
        same = (k == rec["k"]) & np.all(cv_mean == rec["cv_mean"], 1)
        agree += int(same.sum())
        total += len(k)
    assert agree >= 0.97 * total, (agree, total)


def test_auc_matches_roc_auc_score():
    from sklearn.metrics import roc_auc_score
    rng = np.random.default_rng(1)
    for trial in range(300):
        n = int(rng.integers(2, 80))
        y = rng.integers(0, 2, n)
        y[:2] = (0, 1)
        s = rng.integers(0, 6, n) / 5.0 if trial % 2 else rng.random(n)
        ref = roc_auc_score(y, s)
        assert abs(tabular.roc_auc(y, s) - ref) <= 1e-12
        assert abs(T.auc(y, s) - ref) <= 1e-12
    ys, ss = rng.integers(0, 2, (7, 40)), rng.random((7, 40))
    ys[:, :2] = (0, 1)
    np.testing.assert_allclose(tabular.roc_auc(ys, ss), [roc_auc_score(a, b) for a, b in zip(ys, ss)], rtol=0, atol=1e-12)
    with pytest.raises(ValueError):
        tabular.roc_auc(np.ones(5), rng.random(5))


def _fake_metric(x, y, test_x, test_y, cat):
    """A per-sample 'classifier' whose outputs expose what it received: the sum of the standardised test features."""
    out = test_x.sum(1).double().numpy()
    return float(out.mean()), out


def test_harness_windows_selection_keys_and_cache(tmp_path, monkeypatch):
    monkeypatch.setattr(tabular, "RESULTS_DIR", str(tmp_path))
    os.makedirs(tmp_path / "sub", exist_ok=True)
    ds = GOLDEN["datasets"][:2]
    state = torch.get_rng_state()
    r = tabular.evaluate(ds, _fake_metric, 'fake', bptt=GOLDEN["bptt"], eval_position_range=GOLDEN["positions"],
                         device='cpu', max_samples=GOLDEN["max_samples"], save=True, path_interfix='sub')
    assert torch.equal(state, torch.get_rng_state())
    for name, X, y, _ in ds:
        for p in GOLDEN["positions"]:
            gold = GOLDEN["knn"][(name, p)]
            assert torch.equal(r[f'{name}_ys_at_{p}'], gold["ys"].float())  # windows and the seed-13 selection
            eval_xs, eval_ys = T.windows(X, y, GOLDEN["bptt"], GOLDEN["max_samples"])
            pre = eval_xs[:p]
            want = ((eval_xs[p:] - pre.mean(0)) / (pre.std(0) + 1e-6)).sum(-1).double().numpy()
            np.testing.assert_allclose(r[f'{name}_outputs_at_{p}'], want, rtol=1e-5, atol=1e-4)
            assert r[f'{name}_outputs_at_{p}'].shape == gold["ones"].shape
            assert isinstance(r[f'{name}_per_ds_metric_at_{p}'], np.ndarray)
            assert isinstance(r[f'{name}_mean_metric_at_{p}'], float)
        assert os.path.isfile(tmp_path / "sub" / f"results_fake_{name}.npy")
    names, pos = [d[0] for d in ds], GOLDEN["positions"]
    unsaved = {'metric', 'mean_metric'} | {f'mean_metric_at_{p}' for p in pos} | {f'{n}_time' for n in names} | \
        {f'{n}_mean_metric_at_{p}' for n in names for p in pos}
    all_names = [d[0] for d in GOLDEN["datasets"]]
    assert set(GOLDEN["knn_result"]) == {k for k in unsaved if not k.startswith(tuple(names))} | \
        {f'{n}_{k}' for n in all_names for k in ['time'] + [f'mean_metric_at_{p}' for p in pos]}
    assert set(r) == unsaved | {f'{n}_{k}_at_{p}' for n in names for k in ('per_ds_metric', 'outputs', 'ys') for p in pos}
    np.testing.assert_allclose(r['mean_metric'], np.mean([r[f'mean_metric_at_{p}'] for p in GOLDEN["positions"]]))
    again = tabular.evaluate(ds, None, 'fake', bptt=GOLDEN["bptt"], eval_position_range=GOLDEN["positions"],
                             device='cpu', max_samples=GOLDEN["max_samples"], path_interfix='sub')
    for k, v in r.items():
        if k.endswith('_time') or k == 'metric':
            continue
        np.testing.assert_array_equal(np.asarray(again[k]), np.asarray(v))


def test_harness_extend_and_rescale_features(monkeypatch, tmp_path):
    monkeypatch.setattr(tabular, "RESULTS_DIR", str(tmp_path))
    seen = []
    orig = tabular.evaluate_dataset

    def spy(X, y, cat, model, bptt, positions, plot=False, rescale_features=1.0, max_samples=40):
        seen.append((X.shape, rescale_features))
        return orig(X, y, cat, model, bptt, positions, rescale_features=rescale_features, max_samples=max_samples)

    monkeypatch.setattr(tabular, "evaluate_dataset", spy)
    name, X, y, cat = GOLDEN["datasets"][0]
    tabular.evaluate([[name, X, y, cat]], _fake_metric, 'fake', bptt=100, eval_position_range=[30], device='cpu',
                     max_features=60, extend_features=True, rescale_features=True, save=False, max_samples=5)
    assert seen == [((X.shape[0], 60), X.shape[1] / 60)]


def test_dataset_shorter_than_bptt_raises():
    X, y = torch.randn(100, 3), (torch.arange(100) % 2).float()
    with pytest.raises(ValueError):
        tabular.evaluate_position(X, y, [], _fake_metric, 100, 30)


def _context_columns(g, bptt, S):
    """Feature columns where the per-context standardisation goes wrong: standard normal, a constant, integers, large
    offsets with unit and with tiny spread, a spread of 1e-6 around 1, and integers at 1e6."""
    x = torch.randn(bptt, S, 7, generator=g, dtype=torch.float64)
    x[..., 1] = 3.25
    x[..., 2] = torch.randint(-5, 6, (bptt, S), generator=g)
    x[..., 3] = 1e4 + torch.randn(bptt, S, generator=g)
    x[..., 4] = -3e5 + 1e-2 * torch.randn(bptt, S, generator=g)
    x[..., 5] = 1.0 + 1e-6 * torch.randn(bptt, S, generator=g)
    x[..., 6] = 1e6 + torch.randint(0, 3, (bptt, S), generator=g)
    return x.float()


@pytest.mark.parametrize("p", [1, 2, 10, 30, 64, 99])
def test_pfn_contexts_match_the_fp64_oracle_elementwise(p):
    """tabular.pfn_contexts (incremental fp64 statistics from the train prefix) against tabular_oracle.pfn_contexts_ref
    (two-pass fp64 statistics of each context), element by element.  The one fp32 rounding is 2^-24 |x|.  Each side's
    fp64 work rounds ctx - mean and carries its mean's rounding, a few units of 2^-53 (|ctx| + mean |ctx|) before the
    division by std (a sum's rounding scales with the sum of magnitudes, so an integer column whose mean is 0 still
    carries one): where the standardised value is near 0 (a large offset, a tiny spread) that term is the larger one,
    so the bound takes it twice.  A column constant in a context must give exactly 0, and ys must be exact."""
    g = torch.Generator().manual_seed(p)
    bptt, S = 100, 20
    x = _context_columns(g, bptt, S)
    y = (torch.rand(bptt, S, generator=g) < 0.5).float()
    Q, F = bptt - p, x.shape[2]
    for rescale in (1.0, 7 / 60):
        xs, ys = tabular.pfn_contexts(x, y, p, rescale)
        rx, ry = T.pfn_contexts_ref(x, y, p, rescale)
        assert xs.dtype == ys.dtype == torch.float32 and xs.shape == (p + 1, Q * S, F) and ys.shape == (p + 1, Q * S)
        assert torch.equal(ys[:p], ry.float()) and bool((ys[p] == 0).all())
        xd = x.double()
        ctx = torch.cat([xd[:p].unsqueeze(1).expand(p, Q, S, F), xd[p:].unsqueeze(0)], 0).reshape(p + 1, Q * S, F)
        std = ((ctx - ctx.mean(0)) ** 2).sum(0).div(p).sqrt() + 1e-6
        bound = 2.0 ** -24 * rx.abs() + 2 * 2.0 ** -53 * (ctx.abs() + ctx.abs().mean(0)) / std / rescale
        EB.check(f"pfn_contexts p={p} rescale={rescale:.3g}", xs, rx, bound, 1.0)
        flat = (ctx == ctx[:1]).all(0)                                 # columns constant in their context
        assert bool(flat[:, 1].all()) and (p > 2 or bool(flat[:, 2].any()))     # the constant column; integer ties
        assert bool((xs.permute(1, 2, 0)[flat] == 0).all())


NOTEBOOK_BNN_CONFIG = {
    'batch_size': 512, 'bptt': 50, 'dropout': 0.5, 'emsize': 512, 'epochs': 100, 'eval_positions': [10, 20, 40],
    'lr': 1.6421403128751275e-05, 'nhead': 4, 'nhid_factor': 2, 'nlayers': 5, 'num_features': 60,
    'prior_activations': "<class 'torch.nn.modules.activation.Tanh'>",
    'prior_dropout_sampler': {'lambda: 0.0': '<function <lambda> at 0x7f613c1364c0>'},
    'prior_emsize_sampler': {'scaled_beta_sampler_f(2.0, 4.0, 150, 2)': '<function <lambda>.<locals>.<lambda> at 0x7f613c136310>'},
    'prior_is_causal': False,
    'prior_nlayers_sampler': {'lambda: 3': '<function <lambda> at 0x7f613c136790>'},
    'prior_noise_std_gamma_k': 1.8663049257557085, 'prior_noise_std_gamma_theta': 0.05275478076173361,
    'prior_normalize_by_used_features': False,
    'prior_num_features_used_sampler': {'scaled_beta_sampler_f(1.0, 1.6, max_features, 2)': '<function <lambda>.<locals>.<lambda> at 0x7f613c136550>'},
    'prior_order_y': True, 'prior_sigma_gamma_k': 3.6187797729244253, 'prior_sigma_gamma_theta': 0.06773738681062867,
    'prior_type': 'mlp'}
GP_CONFIG = dict(NOTEBOOK_BNN_CONFIG, prior_type='gp', prior_noise=1e-3, prior_outputscale=2.3, prior_lengthscale=1.5e-4,
                 prior_normalize_by_used_features=True, prior_order_y=False)


def test_get_model_builds_the_notebook_bnn_model_with_the_checkpoint_layout():
    model = tabular.get_model(NOTEBOOK_BNN_CONFIG, 'cpu', [30], should_train=False)[2]
    assert [(k, tuple(v.shape)) for k, v in model.state_dict().items()] == GOLDEN["bnn_ckpt_layout"]


@pytest.mark.parametrize("prior_type", ["mlp", "gp", "custom_gp_mix", "gp_mix"])
def test_get_model_passes_the_reference_arguments(monkeypatch, prior_type):
    cfg = dict(GP_CONFIG, prior_type=prior_type, prior_lengthscale_mean=1.0, prior_lengthscale_std_f=0.5,
               prior_outputscale_mean=2.0, prior_outputscale_std_f=0.5, prior_lengthscale_concentration=1.5, prior_nu=2.5,
               prior_outputscale_concentration=0.7, prior_y_minmax_norm=True, prior_noise_concentration=1.1,
               prior_noise_rate=100.0)
    if prior_type == 'mlp':
        cfg = NOTEBOOK_BNN_CONFIG
    calls = []
    monkeypatch.setattr(tabular, "train", lambda *a, **kw: calls.append((a, kw)) or "trained")
    assert tabular.get_model(cfg, 'cpu', [10, 30]) == "trained"
    (args, kw), = calls
    loaders = {'mlp': pfn.priors.mlp.DataLoader, 'gp': pfn.priors.fast_gp.DataLoader,
               'custom_gp_mix': pfn.priors.fast_gp.DataLoader, 'gp_mix': pfn.priors.fast_gp_mix.DataLoader}
    assert args == (loaders[prior_type], tabular.Losses.bce, pfn.encoders.Linear)
    sampler = kw.pop('single_eval_pos_gen')
    assert all(0 <= sampler() <= 30 for _ in range(50))
    extra = kw.pop('extra_prior_kwargs_dict')
    assert kw == dict(emsize=512, nhead=4, y_encoder_generator=pfn.encoders.Linear, pos_encoder_generator=None,
                      batch_size=512, nlayers=5, nhid=1024, epochs=100, warmup_epochs=25, bptt=cfg['bptt'],
                      gpu_device='cpu', dropout=0.5, steps_per_epoch=100, lr=cfg['lr'], verbose=False)
    assert extra['num_features'] == 60 and extra['fuse_x_y'] is False
    assert ('batch_size_per_gp_sample' in extra) == (prior_type == 'mlp')
    if prior_type == 'gp_mix':
        assert extra['hyperparameters'] == tabular.get_gp_mix_prior_hyperparameters(cfg)


def test_hyperparameter_helpers():
    hp = tabular.get_mlp_prior_hyperparameters(NOTEBOOK_BNN_CONFIG)
    assert len(hp) == 17
    assert hp[0] == '<function <lambda> at 0x7f613c136790>' and hp[2] == NOTEBOOK_BNN_CONFIG['prior_activations']
    assert hp[6] is True and hp[8:13] == (None, False, None, None, None) and hp[13:] == (True, False, None, 0.0)
    np.random.seed(0)
    a = hp[3]()
    np.random.seed(0)
    assert a == np.random.gamma(3.6187797729244253, 0.06773738681062867)
    gp = tabular.get_gp_prior_hyperparameters(GP_CONFIG)
    assert gp[0] == 1e-3 and gp[1]() == 2.3 and gp[2]() == 1.5e-4 and gp[3] is True and gp[5:] == (True, False)
    mix = tabular.get_gp_mix_prior_hyperparameters(dict(prior_lengthscale_concentration=1.5, prior_nu=2.5,
                                                        prior_outputscale_concentration=0.7, prior_y_minmax_norm=True,
                                                        prior_noise_concentration=1.1, prior_noise_rate=100.0))
    assert mix == {'lengthscale_concentration': 1.5, 'nu': 2.5, 'outputscale_concentration': 0.7,
                   'categorical_data': True, 'y_minmax_norm': 1.5, 'noise_concentration': 1.1, 'noise_rate': 100.0}
    meta = tabular.get_meta_gp_prior_hyperparameters(dict(GP_CONFIG, prior_lengthscale_mean=0.5, prior_lengthscale_std_f=0.5,
                                                          prior_outputscale_mean=0.5, prior_outputscale_std_f=0.5))
    assert 0 <= meta[1]() <= 1 and 0 <= meta[2]() <= 1 and meta[5:] == (True, False)
    assert tabular.get_default_spec([('a', torch.zeros(5, 7), None, [])], [('b', torch.zeros(5, 9), None, [])]) == (100, [30], 9, 20)


def test_not_provided_baselines_and_dropin():
    for fn in (tabular.logistic_metric, tabular.gp_metric, tabular.bayes_net_metric, tabular.catboost_metric,
               tabular.xgb_metric):
        with pytest.raises(NotImplementedError):
            fn(None, None, None, None, [])
    for cls in (tabular.BayesianModel, tabular.BayesianNNClassifier):
        with pytest.raises(NotImplementedError):
            cls({})
    with pytest.raises(NotImplementedError):
        tabular.evaluate([], _fake_metric, 'x', 100, [30], 'cpu', plot=True)
    pfn.install_dropin()
    assert sys.modules['tabular'] is tabular
