"""Stand-ins for the packages the reference tabular.py (and its datasets/__init__.py) import at module level but the
golden generator never calls: pyro, catboost, xgboost, openml and matplotlib are not installed.  `install()` puts empty
modules with the few names those imports bind into sys.modules.  TEST INFRASTRUCTURE ONLY."""
import sys
import types


class _Placeholder:
    """Any attribute, call or subscript gives another placeholder (PyroModule[nn.Linear], dist.Normal(...), ...)."""

    def __init__(self, *args, **kwargs):
        pass

    def __class_getitem__(cls, item):
        return cls

    def __getattr__(self, name):
        return _Placeholder()

    def __call__(self, *args, **kwargs):
        return _Placeholder()


NAMES = {
    "pyro": [], "pyro.distributions": [], "pyro.nn": ["PyroModule", "PyroSample"],
    "pyro.infer": ["SVI", "Trace_ELBO", "Predictive", "MCMC", "NUTS"], "pyro.infer.autoguide": ["AutoDiagonalNormal"],
    "catboost": ["CatBoostClassifier", "Pool"], "catboost.datasets": ["titanic", "amazon"],
    "xgboost": [], "openml": [], "matplotlib": [], "matplotlib.pyplot": [], "matplotlib.gridspec": [],
}


def install():
    for name, attrs in NAMES.items():
        if name in sys.modules:
            continue
        mod = types.ModuleType(name)
        mod.__path__ = []
        mod.__getattr__ = lambda attr: _Placeholder if not attr.startswith("__") else None
        for a in attrs:
            setattr(mod, a, _Placeholder)
        sys.modules[name] = mod
        parent, _, child = name.rpartition(".")
        if parent:
            setattr(sys.modules[parent], child, mod)
