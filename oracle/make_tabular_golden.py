"""Generate tests/golden/tabular.pt by running the UNMODIFIED reference tabular.py (with its own datasets module) on CPU.

Run where the reference checkout exists, after oracle/build_ref.py:   python oracle/make_tabular_golden.py
pyro, catboost, xgboost, openml and matplotlib are not installed; oracle/ref_stub/tabular_imports.py stands in for them
(tabular.py imports them at module level; nothing recorded here calls them).  sklearn is the real one.

Recorded:
* datasets: seven binary datasets of the reference's local files (get_svmlight, get_biochem, get_heart), capped at 400
  rows, as [name, X fp32, y fp32, []];
* KNN: the reference's evaluate(ds, knn_metric, 'knn', bptt=100, eval_position_range=[10, 30], max_samples=20,
  save=False, overwrite=True) result dict, and per (dataset, position) evaluate_position's per-sample AUCs, outputs and
  ys (uint8 labels; the outputs as the class-1 neighbour count, proba = count / k), plus sklearn's chosen k and CV
  means per sample and the oracle's relative gap (fp32) between the k-th and (k+1)-th distances of every test row
  (near-ties, which sklearn's tree and brute searches order differently);
* PFN: two reference TransformerModels (BCE head, E 128: one head of 128 and two heads of 64) whose weights
  tabular_oracle.seeded_state_dict draws from the recorded seed (a checksum is stored, not the weights), and
  evaluate(ds, model, 'transformer', max_features=60, extend_features=True, rescale_features=True, ...) plus
  evaluate_position's per-sample AUCs;
* the key -> shape list of results/tabular_model_bnn.ckpt.
"""
import contextlib
import importlib.util
import io
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("PFN_REFERENCE_DIR", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "tabular.pt")
BPTT, POSITIONS, MAX_SAMPLES, MAX_FEATURES = 100, [10, 30], 20, 60
sys.path.insert(0, ROOT)
SVMLIGHT = ["australian", "diabetes", "fourclass", "german.numer", "ionosphere_scale"]
PFN_MODELS = {"dh128": dict(E=128, H=1, nhid=256, L=2, seed=31), "dh64": dict(E=128, H=2, nhid=256, L=2, seed=32)}


def load_reference():
    sys.path[:0] = [os.path.join(ROOT, "oracle", "_ref"), REF]
    from oracle.ref_stub import tabular_imports
    tabular_imports.install()
    spec = importlib.util.spec_from_file_location("ref_tabular", os.path.join(REF, "tabular.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_datasets(tab):
    cwd = os.getcwd()
    os.chdir(REF)
    try:
        ds = [[name, *tab.get_svmlight(name)] for name in SVMLIGHT]
        ds += [["biochem", *tab.get_biochem()], ["heart", *tab.get_heart()]]
    finally:
        os.chdir(cwd)
    return [[name, X[:400].float().contiguous(), y[:400].float().contiguous(), []] for name, X, y in ds]


def pfn_model(case):
    import encoders
    import transformer
    from oracle import tabular_oracle as T
    E = case["E"]
    model = transformer.TransformerModel(encoders.Linear(MAX_FEATURES, E), 1, E, case["H"], case["nhid"], case["L"], 0.0,
                                         y_encoder=encoders.Linear(1, E))
    model.load_state_dict(T.seeded_state_dict(model, case["seed"]))
    return model.eval()


def main():
    from oracle import tabular_oracle as T
    warnings.filterwarnings("ignore")
    tab = load_reference()
    ds = load_datasets(tab)
    quiet = contextlib.redirect_stdout(io.StringIO())
    rec = {"datasets": ds, "bptt": BPTT, "positions": POSITIONS, "max_samples": MAX_SAMPLES, "max_features": MAX_FEATURES}

    from sklearn.model_selection import GridSearchCV
    from sklearn.neighbors import KNeighborsClassifier
    with quiet:
        rec["knn_result"] = tab.evaluate(ds, tab.knn_metric, 'knn', bptt=BPTT, eval_position_range=POSITIONS, device='cpu',
                                         max_samples=MAX_SAMPLES, save=False, overwrite=True)
    knn = {}
    for name, X, y, cat in ds:
        for p in POSITIONS:
            with quiet:
                metric, outputs, ys = tab.evaluate_position(X, y, cat, tab.knn_metric, BPTT, p, max_samples=MAX_SAMPLES)
            eval_xs, eval_ys = T.windows(X, y, BPTT, MAX_SAMPLES)
            ks, means = [], []
            for s in range(eval_xs.shape[1]):        # sklearn's own choice on the reference's (fp32) standardisation
                x = eval_xs[:p, s]
                x = (x - x.mean(0)) / (x.std(0) + .000001)
                n = p
                clf = GridSearchCV(KNeighborsClassifier(), {'n_neighbors': np.arange(1, min(6, n - 1))},
                                   cv=min(5, n // 2)).fit(x, eval_ys[:p, s].long())
                ks.append(int(clf.best_params_['n_neighbors']))
                means.append(clf.cv_results_['mean_test_score'])
            _, _, _, gap = T.knn_position_ref(eval_xs, eval_ys, p)
            ks = np.array(ks)
            ones = np.rint(np.asarray(outputs) * ks).astype(np.uint8)     # proba = ones / k exactly
            assert np.array_equal(ones / ks, np.asarray(outputs))
            assert torch.equal(ys, ys.to(torch.uint8).float())
            knn[(name, p)] = dict(metric=np.asarray(metric), ones=ones, ys=ys.to(torch.uint8), k=ks,
                                  cv_mean=np.stack(means), gap=gap.astype(np.float32))
    rec["knn"] = knn

    pfn = {}
    for key, case in PFN_MODELS.items():
        model = pfn_model(case)
        with quiet, torch.no_grad():
            result = tab.evaluate(ds, model, 'transformer', bptt=BPTT, eval_position_range=POSITIONS, device='cpu',
                                  max_features=MAX_FEATURES, extend_features=True, rescale_features=True, save=False,
                                  overwrite=True, max_samples=MAX_SAMPLES)
            per = {}
            for name, X, y, cat in ds:
                Xe = torch.cat([X, torch.zeros(X.shape[0], MAX_FEATURES - X.shape[1])], -1)
                for p in POSITIONS:
                    metric, outputs, ys = tab.evaluate_position(Xe, y, cat, model, BPTT, p,
                                                                rescale_features=X.shape[1] / MAX_FEATURES,
                                                                max_samples=MAX_SAMPLES)
                    per[(name, p)] = dict(metric=np.asarray(metric))
        pfn[key] = dict(case=case, checksum=T.checksum(model.state_dict()), result=result, per=per)
    rec["pfn"] = pfn

    ckpt = torch.load(os.path.join(REF, "results", "tabular_model_bnn.ckpt"), map_location="cpu", weights_only=False)[0]
    rec["bnn_ckpt_layout"] = [(k, tuple(v.shape)) for k, v in ckpt.items()]
    torch.save(rec, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
