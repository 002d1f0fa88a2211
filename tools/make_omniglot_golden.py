"""Write the Omniglot-prior fixture tests/golden/omniglot_prior.pt by running the UNMODIFIED reference loader
(priors/omniglot.py over datasets/omniglotNshot.py and datasets/omniglot.py) over the synthetic tree of
tests/test_gpu_omniglot_prior.py (`synthetic_bank`, written as PNGs to a temporary directory).  Needs PIL and torchvision;
run where a reference checkout exists:

    python tools/make_omniglot_golden.py --reference-dir <reference checkout>

For each (jonas_style, train) the reference's DataLoader (5-way 5-shot, 28 x 28, translations on) yields 2 000 episodes;
every image is decoded to (class, image, rot90 turn, tx, ty) and the file keeps `episode_summary` of them: the share of
episodes that satisfy each structural invariant and the histograms the test compares with the device sampler.

Shims, none of which touches the reference's files: `datasets/*.py` and `priors/omniglot.py` are loaded without their
package `__init__`s (they import openml, catboost and gpytorch); `np.float` / `np.int`, removed in NumPy 1.24, are
restored; and `os.walk` yields sorted entries while the reference builds its dataset, so that its class, character and
image order is the sorted order of the device bank rather than the filesystem's.
"""
import argparse
import importlib.util
import os
import random
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _test_module():
    spec = importlib.util.spec_from_file_location("_pfn_test_omniglot", os.path.join(ROOT, "tests", "test_gpu_omniglot_prior.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def load_reference_omniglot(reference_dir):
    """The reference's priors/omniglot.py as `priors.omniglot`, with `datasets.omniglot` / `datasets.omniglotNshot` loaded
    from the checkout under an empty `datasets` package and the reference's `utils` from oracle/_ref."""
    from oracle import ref_runner
    ref_runner.load()
    for name in ("float", "int"):
        if name not in np.__dict__:
            setattr(np, name, {"float": float, "int": int}[name])
    pkg = types.ModuleType("datasets")
    pkg.__path__ = [os.path.join(reference_dir, "datasets")]
    sys.modules["datasets"] = pkg
    for name in ("omniglot", "omniglotNshot"):
        setattr(pkg, name, _load(f"datasets.{name}", os.path.join(reference_dir, "datasets", f"{name}.py")))
    return _load("priors.omniglot", os.path.join(reference_dir, "priors", "omniglot.py"))


class sorted_walk:
    """os.walk with sorted directories and files, while active."""

    def __enter__(self):
        self.walk = os.walk

        def walk(top, *a, **k):
            for root, dirs, files in self.walk(top, *a, **k):
                dirs.sort()
                yield root, dirs, sorted(files)
        os.walk = walk

    def __exit__(self, *exc):
        os.walk = self.walk
        return False


def reference_summaries(tm, ref, images, alphabets, episodes, batch):
    out = {}
    for jonas, train in tm.CONFIGS:
        seed = 50 + 2 * jonas + train
        random.seed(seed); np.random.seed(seed); torch.manual_seed(seed)
        with sorted_walk():
            dl = ref.DataLoader(num_steps=episodes // batch, batch_size=batch, seq_len=tm.T, num_features=tm.S * tm.S,
                                num_outputs=tm.N_WAY, train=train, translations=True, jonas_style=jonas)
        t0 = time.perf_counter()
        decs, ys, tys = [], [], []
        for (x, y), target_y in dl:
            decs.append(tm.decode_batch(x.numpy(), images))
            ys.append(y.numpy()); tys.append(target_y.numpy())
        dec, y, ty = np.concatenate(decs, 1), np.concatenate(ys, 1), np.concatenate(tys, 1)
        s = tm.episode_summary(dec, y, ty, images, alphabets, jonas, train, train)
        out[(jonas, train)] = s
        print(f"jonas={jonas} train={train}: {dec.shape[1]} episodes in {time.perf_counter() - t0:.1f} s, invariants "
              f"{s['invariants']}", flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference-dir", required=True, help="checkout of the reference repository")
    a = ap.parse_args()
    tm = _test_module()
    images, alphabets = tm.synthetic_bank()
    ref = load_reference_omniglot(os.path.abspath(a.reference_dir))
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        tm.write_tree(tmp, images, alphabets)
        os.chdir(tmp)                      # the reference reads the relative path 'omniglot'
        try:
            out = reference_summaries(tm, ref, images, alphabets, tm.GOLD_EPISODES, 100)
        finally:
            os.chdir(cwd)
    torch.save(out, os.path.join(OUT, "omniglot_prior.pt"))
    print("omniglot fixture written to", OUT)


if __name__ == "__main__":
    main()
