"""Times `tabular.evaluate` at the notebook's shape (TabularEvalSimple.ipynb): bptt 100, eval position 30, 20 samples,
features padded to 60, 37 seeded synthetic datasets of 400 rows.  The PFN has the shipped checkpoint's architecture
(E 512, 4 heads, 5 layers, nhid 1024) with seeded weights.  Prints the device time of the PFN path and of the KNN path
(one pfn_knn_cv launch per dataset) and, when sklearn is importable, the reference-style per-sample GridSearchCV loop
on the host cores for comparison.  Prints the card's name and power limit beside the numbers.

    python tools/time_tabular.py [--datasets 37] [--no-sklearn]
"""
import argparse
import contextlib
import io
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from transformerscandobayesianinference_b200 import encoders, tabular  # noqa: E402
from transformerscandobayesianinference_b200.transformer import TransformerModel  # noqa: E402
from gpu_timing import card, event_times  # noqa: E402


def synthetic_datasets(n, rows=400, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        F = int(torch.randint(4, 60, (1,), generator=g))
        X = torch.randn(rows, F, generator=g)
        w = torch.randn(F, generator=g)
        y = ((X @ w + 0.5 * torch.randn(rows, generator=g)) > 0).float()
        out.append([f"synthetic_{i}", X, y, []])
    return out


def quiet(fn):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--datasets", type=int, default=37)
    ap.add_argument("--no-sklearn", action="store_true")
    args = ap.parse_args()
    print(f"card: {card('time_tabular')}")
    ds = synthetic_datasets(args.datasets)
    torch.manual_seed(0)
    model = TransformerModel(encoders.Linear(60, 512), 1, 512, 4, 1024, 5, 0.5, y_encoder=encoders.Linear(1, 512)).cuda()
    kw = dict(bptt=100, eval_position_range=[30], device='cpu', max_samples=20, save=False, overwrite=True)
    for label, fn in (("pfn", lambda: tabular.evaluate(ds, model, 'transformer', max_features=60, extend_features=True,
                                                       rescale_features=True, **kw)),
                      ("knn", lambda: tabular.evaluate(ds, tabular.knn_metric, 'knn', **kw))):
        secs = event_times(lambda: quiet(fn), 3)    # one warm-up call first: module loads, allocator
        r = quiet(fn)
        print(f"{label}: evaluate over {len(ds)} datasets: best {min(secs):.3f} s, median {np.median(secs):.3f} s "
              f"(mean AUC {r['mean_metric']:.4f})")
    if not args.no_sklearn:
        try:
            from sklearn.model_selection import GridSearchCV
            from sklearn.neighbors import KNeighborsClassifier
        except ImportError:
            print("sklearn not importable: host GridSearchCV loop not timed")
            return
        import warnings
        warnings.filterwarnings("ignore")

        def host_knn(x, y, test_x, test_y, cat):
            n = len(y)
            clf = GridSearchCV(KNeighborsClassifier(), {'n_neighbors': np.arange(1, min(6, n - 1))}, cv=min(5, n // 2))
            clf.fit(x.numpy(), y.long().numpy())
            pred = clf.predict_proba(test_x.numpy())[:, 1]
            return tabular.metric_used(test_y.numpy(), pred), pred
        t0 = time.time()
        quiet(lambda: tabular.evaluate(ds, host_knn, 'knn_host', **kw))
        secs = time.time() - t0
        print(f"knn (sklearn GridSearchCV per sample on {os.cpu_count()} host cores): {secs:.3f} s")


if __name__ == "__main__":
    main()
