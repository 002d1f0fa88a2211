"""Generate tests/golden/regression_baselines.pt by running the UNMODIFIED reference priors/ridge.py evaluate and
priors/gp.py get_batch / evaluate (loaded by oracle/sklearn_priors_ref.py) on the CPU with sklearn.

    python oracle/make_regression_golden.py

Recorded, per case: the inputs (x [T,B,F], y, y_non_noisy [T,B] fp32), the reference's evaluate output on the whole batch
(losses [T] fp64) and, from one evaluate call per dataset, the per-element losses [T, B].
* ridge: alpha in {0, 1e-3, 1} x F in {1, 3, 10}, T = 40, B = 5, inputs from the reference get_batch(noisy_std=.1);
* gp: F in {1, 10} x length scale in {.1, .6}, T = 60, B = 4, inputs from the reference get_batch (sklearn's sample_y),
  both losses (NLL and MSE).  1-D at .6 reaches the regime where torch's GaussianNLLLoss clamps the variance at 1e-6;
* gp_raise: a NaN in x (dataset 2, row 7): the exception the reference raises and the (t, dataset) where it does.
The sklearn and numpy versions that made the file are stored with it.  The reference pins scikit-learn 0.24.2; the
solver paths relied on (Ridge's Cholesky with its SVD fallback, GaussianProcessRegressor's fit / predict / sample_y)
were read from the recorded version only.
"""
import os
import random
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "regression_baselines.pt")

RIDGE_ALPHAS, RIDGE_FS, RIDGE_T, RIDGE_B = (0.0, 1e-3, 1.0), (1, 3, 10), 40, 5
GP_FS, GP_LS, GP_T, GP_B = (1, 10), (.1, .6), 60, 4


def per_dataset(evaluate, x, y, yn, **kw):
    return torch.stack([evaluate(x[:, b:b + 1], y[:, b:b + 1], yn[:, b:b + 1], **kw)[0] for b in range(x.shape[1])], 1)


def main():
    import sklearn
    from oracle import sklearn_priors_ref
    ridge, gp = sklearn_priors_ref.load()
    out = {"sklearn": sklearn.__version__, "numpy": np.__version__, "torch": torch.__version__, "ridge": [], "gp": []}
    n_warn = 0
    for ai, alpha in enumerate(RIDGE_ALPHAS):
        for fi, F in enumerate(RIDGE_FS):
            torch.manual_seed(100 + 10 * ai + fi)
            x, y, yn = ridge.get_batch(RIDGE_B, RIDGE_T, F, noisy_std=.1)
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                losses = ridge.evaluate(x, y, yn, alpha=alpha)[0]
                elem = per_dataset(ridge.evaluate, x, y, yn, alpha=alpha)
            n_warn += len(w)
            out["ridge"].append(dict(alpha=alpha, F=F, x=x, y=y, y_non_noisy=yn, losses=losses.double(), elem=elem.double()))
    for fi, F in enumerate(GP_FS):
        for li, ls in enumerate(GP_LS):
            torch.manual_seed(200 + 10 * fi + li)
            random.seed(300 + 10 * fi + li)
            x, y, yn = gp.get_batch(GP_B, GP_T, F, noisy_std=ls)
            case = dict(F=F, length_scale=ls, x=x, y=y)
            for use_mse in (False, True):
                key = "mse" if use_mse else "nll"
                case[key] = gp.evaluate(x, y, yn, use_mse=use_mse, length_scale=ls)[0].double()
                case[key + "_elem"] = per_dataset(gp.evaluate, x, y, yn, use_mse=use_mse, length_scale=ls).double()
            out["gp"].append(case)
    # where the reference raises: the first (t, dataset) in its loop order, found by growing the sequence
    torch.manual_seed(400)
    x, y = torch.rand(12, 4, 2), torch.randn(12, 4)
    x[7, 2, 1] = float("nan")
    err = None
    try:
        gp.evaluate(x, y, y)
    except Exception as e:          # noqa: BLE001 -- recorded as it is
        err = e
    T_ok = max(T for T in range(2, 13) if _runs(gp, x[:T], y[:T]))
    b_fail = next(b for b in range(4) if not _runs(gp, x[:T_ok + 1, b:b + 1], y[:T_ok + 1, b:b + 1]))
    out["gp_raise"] = dict(x=x, y=y, exception=type(err).__name__, is_value_error=isinstance(err, ValueError),
                           message=str(err), t=T_ok, dataset=b_fail)
    out["ridge_warnings"] = n_warn
    torch.save(out, OUT)
    print(f"wrote {OUT}: {len(out['ridge'])} ridge and {len(out['gp'])} gp cases, sklearn {sklearn.__version__}, "
          f"{n_warn} sklearn warnings in the ridge runs; the reference raises {out['gp_raise']['exception']} at "
          f"t={T_ok}, dataset {b_fail}")


def _runs(gp, x, y):
    try:
        gp.evaluate(x, y, y)
        return True
    except ValueError:
        return False


if __name__ == "__main__":
    main()
