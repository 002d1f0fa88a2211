"""priors.omniglot host logic (no GPU): the image bank against the reference's transform chain, its sorted class order,
the missing-data error, argument validation before any device work, and the shift rule against torchvision."""
import os

import numpy as np
import pytest
import torch

from transformerscandobayesianinference_b200 import _lib as L
from transformerscandobayesianinference_b200.priors import omniglot
from test_gpu_omniglot_prior import shift_image

PIL = pytest.importorskip("PIL")
from PIL import Image  # noqa: E402

# (split, alphabet, characters), created in this (unsorted) order
TREE = [("evaluation", "Zeta", 3), ("background", "Mu", 2), ("evaluation", "Alpha", 2), ("background", "Beta", 4)]


def _write_tree(root, src=40):
    """Small tree of PNGs in modes '1', 'L' and 'RGB'; file names are created in reverse order."""
    rng = np.random.default_rng(1)
    for split, alphabet, n in TREE:
        for c in reversed(range(n)):
            d = os.path.join(root, "omniglot", "processed", f"images_{split}", alphabet, f"character{c + 1:02d}")
            os.makedirs(d)
            for i in reversed(range(20)):
                a = np.full((src, src), 255, np.uint8)
                r, k = rng.integers(0, src - 12, 2)
                a[r:r + 12, k:k + 12] = rng.integers(0, 256, (12, 12))
                mode = ("1", "L", "RGB")[i % 3]
                im = Image.fromarray(a).convert(mode)
                im.save(os.path.join(d, f"{len(alphabet)}{c:02d}_{i + 1:02d}.png"))


def _reference_chain(path, S):
    """datasets/omniglotNshot.py:105-112: open, convert('L'), resize((S, S)), /255., 1 - x (float64), then float32."""
    x = np.reshape(Image.open(path).convert('L').resize((S, S)), (S, S, 1))
    x = np.transpose(x, [2, 0, 1])
    return (1 - x / 255.)[0].astype(np.float32)


@pytest.mark.parametrize("S", [28, 13])
def test_bank_is_the_reference_transform_in_sorted_order(tmp_path, monkeypatch, S):
    _write_tree(str(tmp_path))
    monkeypatch.chdir(tmp_path)
    bank = omniglot.build_bank(S)
    assert bank.images.shape == (11, 20, S, S) and bank.images.dtype == np.uint8
    # sorted (folder, alphabet, character, file): background first
    assert bank.alphabets == [("background", 0, 4), ("background", 4, 2), ("evaluation", 6, 2), ("evaluation", 8, 3)]
    order = [(s, a) for s in omniglot.SPLITS for a in sorted(x[1] for x in TREE if x[0] == s)]
    lut = (1 - np.arange(256) / 255.).astype(np.float32)
    cls = 0
    for split, alphabet in order:
        adir = os.path.join("omniglot", "processed", f"images_{split}", alphabet)
        for ch in sorted(os.listdir(adir)):
            files = sorted(os.listdir(os.path.join(adir, ch)))
            for i, f in enumerate(files):
                ref = _reference_chain(os.path.join(adir, ch, f), S)
                assert np.array_equal(lut[bank.images[cls, i]], ref), (alphabet, ch, f)
            cls += 1
    assert cls == 11
    assert bank.split_alphabets(True) == ([0, 4], [4, 2])
    assert bank.split_alphabets(False) == ([6, 8], [2, 3])
    assert omniglot.load_bank(S) is omniglot.load_bank(S)


def test_missing_data_raises_without_downloading(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    with pytest.raises(FileNotFoundError) as e:
        omniglot.build_bank(28)
    msg = str(e.value)
    for s in ("images_background", "images_evaluation", "images_background.zip", "images_evaluation.zip"):
        assert s in msg
    with pytest.raises(FileNotFoundError):
        omniglot.DataLoader(num_steps=1, batch_size=2, seq_len=26, num_features=784, num_outputs=5)
    assert not os.path.exists(tmp_path / "omniglot")


def test_arguments_are_rejected_before_any_device_work(tmp_path, monkeypatch):
    _write_tree(str(tmp_path))
    monkeypatch.chdir(tmp_path)

    def no_launch(*a, **k):
        raise AssertionError("the kernel was reached")
    monkeypatch.setattr(L, "omniglot_episodes", no_launch)
    kw = dict(num_steps=1, batch_size=2, seq_len=26, num_features=784, num_outputs=5)
    with pytest.raises(AssertionError, match="fusing"):
        omniglot.DataLoader(**dict(kw, fuse_x_y=True))
    with pytest.raises(AssertionError):
        omniglot.DataLoader(**dict(kw, num_features=785))
    with pytest.raises(AssertionError):
        omniglot.DataLoader(**dict(kw, seq_len=25))                        # T != n_way * k_shot + 1
    with pytest.raises(ValueError, match="k_shot"):
        omniglot.DataLoader(**dict(kw, seq_len=5 * 20 + 1))
    with pytest.raises(ValueError, match="num_outputs"):
        omniglot.DataLoader(**dict(kw, num_outputs=65, seq_len=66))
    with pytest.raises(ValueError, match="image side"):
        omniglot.DataLoader(**dict(kw, num_features=106 * 106))
    with pytest.raises(ValueError, match="test pool has 0"):                # classes[1200:] of an 11-class bank
        omniglot.DataLoader(**dict(kw, train=False))
    with pytest.raises(ValueError, match="train pool has 3"):
        omniglot.DataLoader(**dict(kw, num_classes_used=3))
    with pytest.raises(ValueError, match="smallest has 2"):
        omniglot.DataLoader(**dict(kw, jonas_style=True, num_outputs=3, seq_len=7))
    with pytest.raises(ValueError, match="batch_size"):
        omniglot.DataLoader(**dict(kw, batch_size=0))
    dl = omniglot.DataLoader(**dict(kw, jonas_style=True, num_outputs=2, seq_len=11))
    assert (dl.num_features, dl.num_outputs, dl.fuse_x_y, len(dl)) == (784, 2, False, 1)
    assert (dl.desc.T, dl.desc.n_way, dl.desc.k_shot, dl.desc.n_alpha, dl.desc.alpha_min) == (11, 2, 5, 2, 2)
    d = omniglot.DataLoader(**dict(kw, num_outputs=3, seq_len=7)).desc
    assert (d.pool_lo, d.pool_n, d.translate, d.jonas) == (0, 11, 1, 0)
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            iter(dl)


def test_dropin_registers_priors_omniglot():
    import sys
    import transformerscandobayesianinference_b200 as pfn
    saved = {k: sys.modules.get(k) for k in list(sys.modules) if k.split(".")[0] in pfn._DROPIN_MODULES}
    try:
        pfn.install_dropin()
        assert sys.modules["priors.omniglot"] is omniglot
        assert sys.modules["priors"].omniglot is omniglot
    finally:
        for k in [k for k in list(sys.modules) if k.split(".")[0] in pfn._DROPIN_MODULES]:
            del sys.modules[k]
        sys.modules.update({k: v for k, v in saved.items() if v is not None})


@pytest.mark.parametrize("size", [28, 13, 9])
def test_shift_rule_is_torchvisions_nearest_affine(size):
    tv = pytest.importorskip("torchvision.transforms.functional")
    from torchvision.transforms import InterpolationMode
    rng = np.random.default_rng(size)
    img = rng.random((size, size)).astype(np.float32)
    for tx in range(-size, size + 1, 1 if size < 20 else 3):
        for ty in range(-size, size + 1, 1 if size < 20 else 3):
            ref = tv.affine(torch.from_numpy(img).unsqueeze(0), angle=0.0, translate=[tx, ty], scale=1.0,
                            interpolation=InterpolationMode.NEAREST, shear=[0.0, 0.0], fill=0.).squeeze(0).numpy()
            assert np.array_equal(shift_image(img, tx, ty), ref), (tx, ty)
