"""Ridge baseline, exact GP and binarized priors, host side (no GPU): the fp64 oracle of csrc/regression_baselines.cu
against the unmodified reference's results (tests/golden/regression_baselines.pt, made by
oracle/make_regression_golden.py) and numpy's lstsq, the C-ABI argument checks made before any CUDA call, and the
Python modules' imports and drop-in registration."""
import ctypes
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import regression_baselines_oracle as O
from transformerscandobayesianinference_b200 import _lib as L

GOLDEN = torch.load("tests/golden/regression_baselines.pt", weights_only=False)


@pytest.mark.parametrize("case", range(len(GOLDEN["ridge"])))
def test_ridge_oracle_matches_the_reference(case):
    c = GOLDEN["ridge"][case]
    x, y, yn = c["x"].numpy(), c["y"].numpy(), c["y_non_noisy"].numpy()
    T, B, F = x.shape
    # alpha = 0 on rank-deficient prefixes depends on rounding inside sklearn itself: compared from t = F + 2 on
    t0 = 1 if c["alpha"] > 0 else F + 2
    for b in range(B):
        _, sq, info = O.ridge_prefix_ref(x[:, b], y[:, b], yn[:, b], c["alpha"])
        ref = c["elem"][:, b].numpy()
        gap = np.abs(np.sqrt(ref[t0:]) - np.sqrt(sq[t0:]))          # |err| differences bound the prediction's
        assert np.all(gap <= O.ridge_bound(info)[t0:]), (b, gap.max())
    batch = np.mean([O.ridge_prefix_ref(x[:, b], y[:, b], yn[:, b], c["alpha"])[1] for b in range(B)], 0)
    np.testing.assert_allclose(batch[t0:], c["losses"].numpy()[t0:], rtol=1e-9, atol=1e-15)


@pytest.mark.parametrize("F", [3, 10])
def test_ridge_oracle_is_the_min_norm_lstsq_on_rank_deficient_prefixes(F):
    rng = np.random.default_rng(F)
    x, y = rng.random((F + 2, F)), rng.normal(size=F + 2)
    for t in range(1, F + 1):                                       # centred rank <= t - 1 < F
        _, sq, _ = O.ridge_prefix_ref(x[:t + 1], y[:t + 1], y[:t + 1], 0.0)
        Xc, yc = x[:t] - x[:t].mean(0), y[:t] - y[:t].mean()
        w = np.linalg.lstsq(Xc, yc, rcond=None)[0]
        pred = y[:t].mean() + (x[t] - x[:t].mean(0)) @ w
        assert abs(np.sqrt(sq[t]) - abs(y[t] - pred)) <= 1e-12


@pytest.mark.parametrize("case", range(len(GOLDEN["gp"])))
@pytest.mark.parametrize("use_mse", [False, True])
def test_gp_oracle_matches_the_reference(case, use_mse):
    c = GOLDEN["gp"][case]
    x, y = c["x"].numpy(), c["y"].numpy()
    key = "mse" if use_mse else "nll"
    for b in range(x.shape[1]):
        m, v, status, info = O.exact_gp_ref(x[:, b], y[:, b], c["length_scale"])
        assert status == 0
        loss = O.gp_losses(m, v, y[:, b], use_mse)
        bm, bv = O.exact_gp_bound(info)
        gap = np.abs(loss[1:] - c[key + "_elem"][1:, b].numpy())
        assert np.all(gap <= O.gp_loss_bound(m, v, y[:, b], bm, bv, use_mse)[1:]), (b, gap.max())


def test_gp_nll_reaches_the_variance_clamp():
    c = next(c for c in GOLDEN["gp"] if c["F"] == 1 and c["length_scale"] == .6)
    clamp = 0.5 * np.log(1e-6) + 0.5 * np.log(2 * np.pi)
    assert abs(float(c["nll"][-1]) - clamp) < 1e-4
    m, v, _, _ = O.exact_gp_ref(c["x"][:, 0].numpy(), c["y"][:, 0].numpy(), .6)
    assert v[-1] < 1e-6 and abs(O.gp_losses(m, v, c["y"][:, 0].numpy())[-1] - clamp) < 1e-4


def test_the_reference_raise_case_is_recorded():
    r = GOLDEN["gp_raise"]
    assert r["is_value_error"] and (r["t"], r["dataset"]) == (7, 2)


def test_pivoted_factor_oracle_reproduces_a_singular_kernel():
    x = np.random.default_rng(0).random((128, 1)).astype(np.float32)
    G, perm, r = O.pivoted_cholesky_ref(x, .6)
    K = O.rbf_matrix(x, x, .6)
    assert r < 40 and np.abs(G @ G.T - K).max() <= 1e-12
    assert np.all(np.triu(G[perm], 1) == 0)


def _ridge_desc(B=2, T=8, F=3, alpha=0.0):
    d = L.RidgePrefixDesc()
    d.B, d.T, d.F, d.alpha = B, T, F, alpha
    for name in ("x", "y", "target", "pred", "sq_err"):
        setattr(d, name, 16)             # never dereferenced: the checks fail first
    return d


def _gp_desc(B=2, T=8, F=1, mode=L.EXACT_GP_EVALUATE, ls=.6, alpha=1e-10):
    d = L.ExactGpDesc()
    d.B, d.T, d.F, d.mode, d.length_scale, d.alpha = B, T, F, mode, ls, alpha
    for name in ("x", "y", "z", "mean", "var", "status", "sample", "rank"):
        setattr(d, name, 16)
    return d


@pytest.mark.parametrize("kw, msg", [
    (dict(F=65), b"F=65 exceeds 64"),
    (dict(B=0), b"empty problem"),
    (dict(alpha=-1.0), b"must be finite and >= 0"),
    (dict(alpha=float("inf")), b"must be finite and >= 0"),
])
def test_ridge_cabi_rejects_bad_arguments_before_any_cuda_call(kw, msg):
    lib = L.load()
    assert lib.pfn_ridge_prefix(ctypes.byref(_ridge_desc(**kw)), None) != 0
    assert msg in lib.pfn_last_error()


@pytest.mark.parametrize("kw, msg", [
    (dict(T=129), b"T=129 exceeds 128"),
    (dict(F=0), b"empty problem"),
    (dict(ls=0.0), b"length_scale=0 must be finite and > 0"),
    (dict(mode=2), b"unknown mode 2"),
    (dict(alpha=-1.0), b"alpha=-1 must be finite"),
])
def test_exact_gp_cabi_rejects_bad_arguments_before_any_cuda_call(kw, msg):
    lib = L.load()
    assert lib.pfn_exact_gp(ctypes.byref(_gp_desc(**kw)), None) != 0
    assert msg in lib.pfn_last_error()


def test_exact_gp_cabi_requires_the_outputs_of_its_mode():
    lib = L.load()
    d = _gp_desc(mode=L.EXACT_GP_SAMPLE)
    d.rank = None
    assert lib.pfn_exact_gp(ctypes.byref(d), None) != 0 and b"sample needs" in lib.pfn_last_error()


def test_python_argument_checks_on_the_host():
    from transformerscandobayesianinference_b200.priors import gp, ridge
    x = torch.rand(129, 2, 1)
    with pytest.raises(ValueError, match="129 exceeds 128"):
        gp.evaluate(x, x[..., 0], x[..., 0])
    with pytest.raises(ValueError, match="129 exceeds 128"):
        gp.get_batch(2, 129, 1)
    with pytest.raises(ValueError, match="alpha"):
        ridge.evaluate(x[:5], x[:5, :, 0], x[:5, :, 0], alpha=-1.)
    with pytest.raises(ValueError, match="65 features"):
        ridge.evaluate(torch.rand(5, 2, 65), x[:5, :, 0], x[:5, :, 0])


def test_importing_priors_does_not_import_sklearn():
    code = ("import sys; from transformerscandobayesianinference_b200 import priors; "
            "assert priors.gp and priors.binarized_regression and priors.ridge.evaluate; "
            "print(sorted(m for m in sys.modules if m.split('.')[0] in ('sklearn', 'gpytorch', 'pyro')))")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True)
    assert out.stdout.strip() == "[]"


def test_install_dropin_registers_the_sklearn_priors():
    import transformerscandobayesianinference_b200 as pfn
    saved = dict(sys.modules)
    try:
        pfn.install_dropin()
        import priors
        import priors.binarized_regression as BR
        import priors.gp as G
        import priors.ridge as R
        assert G is pfn.priors.gp and R is pfn.priors.ridge and BR is pfn.priors.binarized_regression
        assert priors.gp is G and G.length_scale_sampling_gp == .6
        for dl in (G.DataLoader, R.DataLoader, BR.Binarized_fast_gp_dataloader, BR.Binarized_fast_gp_mix_dataloader):
            assert dl.num_outputs == 1
        assert callable(BR.regression_prior_to_binary) and callable(R.evaluate) and callable(G.evaluate)
    finally:
        for k in set(sys.modules) - set(saved):
            del sys.modules[k]


def test_labels_are_formed_at_once_and_again_after_pending_checks():
    from transformerscandobayesianinference_b200.priors.utils import _Deferred, again_after_deferred_checks
    calls = []
    again_after_deferred_checks(lambda: calls.append("now"))
    assert calls == ["now"]
    _Deferred.active = True
    try:
        again_after_deferred_checks(lambda: calls.append("no pending check"))
        assert _Deferred.collect() == [] and calls[-1] == "no pending check"
        _Deferred.pending.append(lambda: calls.append("check"))
        again_after_deferred_checks(lambda: calls.append("label"))
        assert calls[-1] == "label"
        for chk in _Deferred.collect():
            chk()
    finally:
        _Deferred.active = False
    assert calls[-3:] == ["label", "check", "label"]
