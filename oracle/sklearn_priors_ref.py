"""The reference's sklearn-backed priors, priors/ridge.py and priors/gp.py, UNMODIFIED, for the golden generator
(oracle/make_regression_golden.py) and tools/time_regression_baselines.py.  TEST / BASELINE INFRASTRUCTURE ONLY.

    python oracle/sklearn_priors_ref.py      # or __graft_entry__.build()

`vendor()` copies the two files into oracle/_ref/sklearn_priors/ (git-ignored) where the reference checkout exists.
`load()` imports them as the package `ref_sklearn_priors` whose `utils` is a stand-in: the reference's priors/utils.py
imports matplotlib at module level, and the two modules take only `get_batch_to_dataloader` from it, to build loader
classes that nothing here uses.  The reference's priors/__init__.py (which imports gpytorch and pyro) is not run.
"""
import importlib
import os
import shutil
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PFN_REFERENCE_DIR", "/root/reference")
DST = os.path.join(HERE, "_ref", "sklearn_priors")
FILES = ["ridge.py", "gp.py"]
PKG = "ref_sklearn_priors"


def vendor(verbose=True):
    """Returns True if oracle/_ref/sklearn_priors is (now) present."""
    if not os.path.isdir(REF):
        return os.path.isdir(DST)
    os.makedirs(DST, exist_ok=True)
    for f in FILES:
        shutil.copyfile(os.path.join(REF, "priors", f), os.path.join(DST, f))
    if verbose:
        print(f"[oracle/sklearn_priors_ref] vendored priors/{{{','.join(FILES)}}} into {DST}")
    return True


def load(src=None):
    """(ridge, gp): the reference modules from `src` (default: the vendored copy, else the reference checkout)."""
    src = src or (DST if os.path.isdir(DST) else os.path.join(REF, "priors"))
    if PKG not in sys.modules:
        pkg = types.ModuleType(PKG)
        pkg.__path__ = [src]
        utils = types.ModuleType(PKG + ".utils")

        def get_batch_to_dataloader(get_batch_method_):
            return type("DL", (), {"get_batch_method": staticmethod(get_batch_method_)})

        utils.get_batch_to_dataloader = get_batch_to_dataloader
        sys.modules[PKG], sys.modules[PKG + ".utils"] = pkg, utils
    return importlib.import_module(PKG + ".ridge"), importlib.import_module(PKG + ".gp")


if __name__ == "__main__":
    sys.exit(0 if vendor() else 1)
