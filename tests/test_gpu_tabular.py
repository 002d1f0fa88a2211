"""The tabular evaluation on the H100: the PFN path (one forward pass per (dataset, eval position)) against the fp64
oracle and the reference's goldens, and the KNN kernel (csrc/knn_cv.cu) against the oracle and sklearn's recorded
choices (tests/golden/tabular.pt, written by oracle/make_tabular_golden.py)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from transformerscandobayesianinference_b200 import _lib as L, encoders, tabular  # noqa: E402
from transformerscandobayesianinference_b200.transformer import TransformerModel  # noqa: E402
from oracle import pfn_oracle as O, tabular_oracle as T  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = torch.load(os.path.join(ROOT, "tests", "golden", "tabular.pt"), weights_only=False)
BPTT, POS, NS, MF = GOLDEN["bptt"], GOLDEN["positions"], GOLDEN["max_samples"], GOLDEN["max_features"]


def _model(key, precision):
    rec = GOLDEN["pfn"][key]
    c = rec["case"]
    m = TransformerModel(encoders.Linear(MF, c["E"]), 1, c["E"], c["H"], c["nhid"], c["L"], 0.0,
                         y_encoder=encoders.Linear(1, c["E"]))
    sd = T.seeded_state_dict(m, c["seed"])
    assert T.checksum(sd) == rec["checksum"]          # the weights the reference ran with
    m.load_state_dict(sd)
    m.precision = precision
    return m.cuda(), O.params_from_state_dict(sd, c["L"]), c["H"]


def _extended(X):
    return torch.cat([X, torch.zeros(X.shape[0], MF - X.shape[1])], -1), X.shape[1] / MF


@pytest.mark.parametrize("key", ["dh128", "dh64"])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_pfn_outputs_match_the_fp64_oracle_and_the_reference_aucs(key, precision):
    model, P, H = _model(key, precision)
    for name, X, y, cat in GOLDEN["datasets"]:
        Xe, rescale = _extended(X)
        for p in POS:
            metric, outputs, ys = tabular.evaluate_position(Xe, y, cat, model, BPTT, p, rescale_features=rescale,
                                                            max_samples=NS)
            eval_xs, eval_ys = T.windows(Xe, y, BPTT, NS)
            ref = T.pfn_outputs_ref(P, H, eval_xs, eval_ys, p, rescale)
            err = np.abs(outputs - ref)
            if precision == "fp32":
                bound = 1e-4 * np.abs(ref) + 1e-6
                assert (err <= bound).all(), (name, p, err.max())
            else:
                bound = 2e-2 * np.maximum(np.abs(ref), 0.05)
                assert (err <= bound).all(), (name, p, err.max())
            b = float(bound.max())
            gold = GOLDEN["pfn"][key]["per"][(name, p)]
            for s in range(outputs.shape[1]):
                lo, hi = T.auc_interval(ys[:, s].numpy(), ref[:, s], b)
                assert lo - 1e-12 <= metric[s] <= hi + 1e-12, (name, p, s)       # 1e-12: rounding of the quotient
                if precision == "fp32":
                    lo, hi = T.auc_interval(ys[:, s].numpy(), ref[:, s], max(b, 1e-4))
                    assert lo - 1e-12 <= gold["metric"][s] <= hi + 1e-12, (name, p, s)
            lo, hi = T.auc_interval(ys.flatten().numpy(), ref.flatten(), b)
            assert lo - 1e-12 <= tabular.metric_used(ys.flatten(), outputs.flatten()) <= hi + 1e-12


def test_pfn_one_forward_pass_per_dataset_and_position():
    model, _, _ = _model("dh128", "bf16")
    name, X, y, cat = GOLDEN["datasets"][0]
    Xe, rescale = _extended(X)
    p = 30
    eval_xs, eval_ys = T.windows(Xe, y, BPTT, NS)
    xs, ys = tabular.pfn_contexts(eval_xs.cuda(), eval_ys.cuda(), p, rescale)
    with torch.no_grad():
        L.reset_launch_count()
        model((xs, ys), single_eval_pos=p)
        one = L.launch_count()
        L.reset_launch_count()
        tabular.evaluate_position(Xe, y, cat, model, BPTT, p, rescale_features=rescale, max_samples=NS)
        assert L.launch_count() == one


def test_pfn_full_size_shape_matches_fp64_oracle():
    """The checkpoint's architecture at the notebook's batch: 1 400 contexts of 31 tokens (the oracle runs on the host)."""
    torch.manual_seed(0)
    E, H, nl, F = 512, 4, 5, 60
    model = TransformerModel(encoders.Linear(F, E), 1, E, H, 2 * E, nl, 0.0, y_encoder=encoders.Linear(1, E))
    with torch.no_grad():
        for layer in model.transformer_encoder.layers:
            layer.linear2.weight.normal_(0, 0.02)
            layer.self_attn.out_proj.weight.normal_(0, 0.02)
    model.precision = "fp32"
    model.cuda()
    S, p = 20, 30
    X = torch.randn(100 + S, F)
    y = (torch.rand(100 + S) < 0.5).float()
    _, outputs, _ = tabular.evaluate_position(X, y, [], model, 100, p, max_samples=S)
    assert outputs.shape == (70, S)                          # 1 400 contexts of 31 tokens
    eval_xs, eval_ys = T.windows(X, y, 100, S)
    xs, ys = T.pfn_contexts_ref(eval_xs, eval_ys, p)
    ys = torch.cat([ys, torch.zeros(1, ys.shape[1], dtype=ys.dtype)], 0)
    P = O.params_from_state_dict(model.state_dict(), nl)
    ref = torch.sigmoid(O.transformer_forward_ref(P, xs, ys, p, H)[0, :, 0]).reshape(70, S).numpy()
    assert (np.abs(outputs - ref) <= 1e-4 * np.abs(ref) + 1e-6).all()


def test_knn_matches_oracle_and_goldens():
    for name, X, y, cat in GOLDEN["datasets"]:
        for p in POS:
            gold = GOLDEN["knn"][(name, p)]
            eval_xs, eval_ys = T.windows(X, y, BPTT, NS)
            proba, k, cv_mean = tabular.knn_cv(tabular.standardize_by_prefix(eval_xs, p), eval_ys[:p])
            r_proba, r_k, r_mean, gap = T.knn_position_ref(eval_xs, eval_ys, p)
            np.testing.assert_array_equal(k.cpu().numpy(), r_k)                  # the oracle, bit for bit
            np.testing.assert_array_equal(cv_mean.cpu().numpy(), r_mean)
            np.testing.assert_array_equal(proba.cpu().numpy(), r_proba)
            # against sklearn on the reference's own standardisation: equal except across near-ties.  The reference
            # standardises in fp32, which moves distances by ~1e-7 relative, so a gap under 1e-5 counts as a near-tie.
            same = (k.cpu().numpy() == gold["k"]) & np.all(cv_mean.cpu().numpy() == gold["cv_mean"], 1)
            clear = same & np.all(gap >= 1e-5, 0)
            np.testing.assert_array_equal(proba.cpu().numpy()[:, clear], (gold["ones"] / gold["k"])[:, clear])
            metric, outputs, _ = tabular.evaluate_position(X, y, cat, tabular.knn_metric, BPTT, p, max_samples=NS)
            np.testing.assert_array_equal(outputs, proba.cpu().numpy())
            np.testing.assert_allclose(metric[clear], gold["metric"][clear], rtol=0, atol=1e-12)   # AUC quotient rounding
            assert same.mean() >= 0.9, (name, p, same.mean())


def test_knn_one_launch_per_dataset_and_position_and_single_problem_agrees():
    name, X, y, cat = GOLDEN["datasets"][0]
    L.reset_launch_count()
    r = tabular.evaluate([[name, X, y, cat]], tabular.knn_metric, 'knn', bptt=BPTT, eval_position_range=POS,
                         device='cpu', max_samples=NS, save=False, overwrite=True)
    assert L.launch_count() == len(POS)
    assert abs(r[f'{name}_mean_metric_at_30'] - GOLDEN["knn_result"][f'{name}_mean_metric_at_30']) < 0.05
    eval_xs, eval_ys = T.windows(X, y, BPTT, NS)
    xs = tabular.standardize_by_prefix(eval_xs, 30)
    batched, _, _ = tabular.knn_cv(xs, eval_ys[:30])
    for s in range(3):
        metric, pred = tabular.knn_metric(xs[:30, s], eval_ys[:30, s], xs[30:, s], eval_ys[30:, s], [])
        np.testing.assert_array_equal(pred, batched[:, s].cpu().numpy())


def test_knn_and_metric_errors():
    x = torch.randn(40, 2, 3)
    y = (torch.arange(30) % 2).float().reshape(30, 1).repeat(1, 2)
    with pytest.raises(ValueError, match="one class"):
        tabular.knn_cv(x, torch.zeros(30, 2))
    bad = y.clone()
    bad[3, 1] = 2.0
    with pytest.raises(ValueError, match="0 or 1"):
        tabular.knn_cv(x, bad)
    few = torch.zeros(30, 2)
    few[:2] = 1.0                    # 2 and 28 members, 5 folds: sklearn accepts it (one class has enough members)
    tabular.knn_cv(x, few)
    with pytest.raises(ValueError):
        tabular.knn_cv(torch.randn(6, 1, 2), torch.tensor([[0.], [1.], [0.]]))      # n = 3 < 4
    with pytest.raises(ValueError):
        tabular.metric_used(np.ones(4), np.arange(4.0))
    with pytest.raises(ValueError):
        tabular.evaluate_position(torch.randn(100, 3), torch.ones(100), [], tabular.knn_metric, 100, 30)

