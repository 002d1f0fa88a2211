"""`priors.omniglot` (reference priors/omniglot.py, datasets/omniglotNshot.py, datasets/omniglot.py): few-shot episodes of
Omniglot characters, the fine-tuning and evaluation data of the FewShotOmniglot notebook.

Image bank (omniglotNshot.py:98-134, omniglot.py:38-56,115-133).  Every PNG under
`omniglot/processed/images_{background,evaluation}/<alphabet>/<character>/` (relative to the working directory) goes
through `Image.open(f).convert('L')` and `.resize((S, S))` with Pillow's default filter.  The reference then forms
`1 - x / 255.` in float64 and casts to float32; here the bank keeps the uint8 pixels, [1623, 20, S, S] (about 25 MB at
S = 28), resident on the device, and the kernel forms `(float)(1.0 - v / 255.0)`, which is bit-equal.  It is built once
per process, data directory and image side.  Nothing is downloaded: missing folders raise FileNotFoundError.

Known difference: the reference orders classes, characters and images in `os.walk` order, which depends on the filesystem.
Here they are sorted by (folder, alphabet, character, file name), so the background alphabets come first and the default
1200-class train split is the 964 background characters plus the first 236 evaluation characters.

Default episode (OmniglotNShot.load_data_cache, omniglotNshot.py:172-230): n_way distinct classes of the pool (train:
classes[:num_classes_used], test: classes[1200:]), class j labelled j; per class k_shot + 1 distinct images of its 20 and
one np.rot90 turn k in {0..3} shared by them (also in test mode); the n_way * k_shot support images in a uniformly random
order; the query (priors/omniglot.py:61 keeps the first of the shuffled queries) is a uniformly chosen class's last drawn
image.

Jonas episode (OmniglotNShotJonas.next, omniglotNshot.py:32-77): a uniform alphabet of the split (train: the background
alphabets, test: the evaluation ones); its first n_way characters in a random order, character j labelled j; the support
class-major, unrotated.  Train: k_shot + 1 distinct images per class; test: images 0..k_shot-1 in a random order as
support and a query image uniform on k_shot..19.  The query class is uniform.

Batch (priors/omniglot.py:59-72): ((x [T, B, S²] fp32, y [T, B] int64), target_y), T = n_way * k_shot + 1, the query in the
last row, target_y = y with -100 in every row but the last.  With `train and translations` every image is shifted after
its rotation by integers (tx, ty) drawn uniformly from [-c0, S-1-c1] x [-r0, S-1-r1], (r0..r1, c0..c1) being the bounding
box of its nonzero pixels, with NEAREST sampling and fill 0 (priors/omniglot.py:12-34), so the ink stays inside.  An image
without ink is left unshifted (the reference raises IndexError there).

A batch is one launch of csrc/omniglot_prior.cu writing x, y and target_y on the current CUDA device.  Its random numbers
are counter-based hashes of one seed per batch drawn from torch's CPU generator: no device sync, and a batch is
reproducible under `torch.manual_seed`.  The distribution is the reference's; numpy's and Python's random streams are not
replayed.  There is no CPU fallback.
"""
import math
import os

import numpy as np
import torch

from .. import _lib as L
from ..utils import set_locals_in_self
from .prior import PriorDataLoader

SPLITS = ("background", "evaluation")
TEST_CLASSES_FROM = 1200          # OmniglotNShot: x_test = x[1200:], hard-coded (omniglotNshot.py:132)


class Bank:
    """uint8 images [n_classes, 20, S, S] in class order, and the alphabets as (split, first class, characters)."""

    def __init__(self, images, alphabets):
        self.images = np.ascontiguousarray(images, dtype=np.uint8)
        assert self.images.ndim == 4 and self.images.shape[1] == L.OMNIGLOT_IMAGES and self.images.shape[2] == self.images.shape[3]
        self.alphabets = [(s, int(f), int(n)) for s, f, n in alphabets]
        self.S = self.images.shape[2]
        self.n_classes = self.images.shape[0]
        self._device = {}

    def split_alphabets(self, train):
        """(first classes, sizes) of the alphabets that serve `train` (background) or test (evaluation) in Jonas mode."""
        split = SPLITS[0] if train else SPLITS[1]
        al = [(f, n) for s, f, n in self.alphabets if s == split]
        return [f for f, _ in al], [n for _, n in al]

    def on_device(self, device, train):
        """(bank, alpha_start of the split) as device tensors, uploaded once per device."""
        key = torch.device(device)
        if key not in self._device:
            bank = torch.from_numpy(self.images).to(key)
            starts = {t: torch.tensor(self.split_alphabets(t)[0] or [0], dtype=torch.int32, device=key) for t in (True, False)}
            self._device[key] = (bank, starts)
        bank, starts = self._device[key]
        return bank, starts[bool(train)]


def build_bank(S, root='omniglot'):
    """The reference's transform chain over the extracted tree under `root`, in sorted order."""
    dirs = [os.path.join(root, 'processed', f'images_{s}') for s in SPLITS]
    if not all(os.path.isdir(d) for d in dirs):
        raise FileNotFoundError(
            f"priors.omniglot: the Omniglot images are missing: expected the directories {dirs[0]!r} and {dirs[1]!r} "
            f"(relative to {os.getcwd()!r}), i.e. images_background.zip and images_evaluation.zip extracted under "
            f"{os.path.join(root, 'processed')!r}.  Nothing is downloaded.")
    from PIL import Image

    def subdirs(d):
        return sorted(e for e in os.listdir(d) if os.path.isdir(os.path.join(d, e)))

    images, alphabets = [], []
    for split, d in zip(SPLITS, dirs):
        for alphabet in subdirs(d):
            first = len(images)
            for character in subdirs(os.path.join(d, alphabet)):
                cdir = os.path.join(d, alphabet, character)
                files = sorted(f for f in os.listdir(cdir) if f.endswith("png"))
                if len(files) != L.OMNIGLOT_IMAGES:
                    raise ValueError(f"priors.omniglot: {cdir} holds {len(files)} images, expected {L.OMNIGLOT_IMAGES}")
                imgs = []
                for f in files:
                    with Image.open(os.path.join(cdir, f)) as im:
                        imgs.append(np.asarray(im.convert('L').resize((S, S)), dtype=np.uint8))
                images.append(np.stack(imgs))
            if len(images) > first:
                alphabets.append((split, first, len(images) - first))
    if not images:
        raise FileNotFoundError(f"priors.omniglot: no character folders under {dirs[0]!r} or {dirs[1]!r}")
    return Bank(np.stack(images), alphabets)


_BANKS = {}


def load_bank(S, root='omniglot'):
    """`build_bank`, once per process, data directory and image side."""
    key = (os.path.realpath(root), S)
    if key not in _BANKS:
        _BANKS[key] = build_bank(S, root)
    return _BANKS[key]


def episode_shape(seq_len, num_features, num_outputs):
    """-> (S, n_way, k_shot), with the reference's assertions (priors/omniglot.py:41-44) and this sampler's limits."""
    S = math.isqrt(num_features)
    assert S * S == num_features
    assert ((seq_len - 1) // num_outputs) * num_outputs == seq_len - 1
    k_shot = (seq_len - 1) // num_outputs
    if k_shot + 1 > L.OMNIGLOT_IMAGES:
        raise ValueError(f"priors.omniglot: seq_len={seq_len} with num_outputs={num_outputs} needs k_shot + 1 = {k_shot + 1} "
                         f"images per class; a class has {L.OMNIGLOT_IMAGES}")
    if not 1 <= num_outputs <= L.OMNIGLOT_MAX_WAY:
        raise ValueError(f"priors.omniglot: num_outputs={num_outputs} outside [1, {L.OMNIGLOT_MAX_WAY}]")
    if not 1 <= S <= L.OMNIGLOT_MAX_SIDE:
        raise ValueError(f"priors.omniglot: image side {S} outside [1, {L.OMNIGLOT_MAX_SIDE}] "
                         f"(num_features = side^2 <= {L.OMNIGLOT_MAX_SIDE ** 2})")
    return S, num_outputs, k_shot


def episode_desc(bank, batch_size, n_way, k_shot, train=True, jonas_style=False, translations=True, num_classes_used=1200):
    """The kernel's descriptor, every argument checked against the bank on the host."""
    if batch_size < 1:
        raise ValueError(f"priors.omniglot: batch_size={batch_size} must be >= 1")
    d = L.OmniglotDesc()
    d.S, d.n_classes, d.B = bank.S, bank.n_classes, batch_size
    d.n_way, d.k_shot, d.T = n_way, k_shot, n_way * k_shot + 1
    d.jonas, d.train, d.translate = int(bool(jonas_style)), int(bool(train)), int(bool(train and translations))
    if jonas_style:
        starts, sizes = bank.split_alphabets(train)
        split = SPLITS[0] if train else SPLITS[1]
        if not sizes:
            raise ValueError(f"priors.omniglot: no {split} alphabets in the bank")
        if n_way > min(sizes):
            raise ValueError(f"priors.omniglot: {n_way}-way Jonas episodes need {n_way} characters in every {split} alphabet; "
                             f"the smallest has {min(sizes)}")
        d.n_alpha, d.alpha_min = len(sizes), min(sizes)
    else:
        lo, hi = (0, min(num_classes_used, bank.n_classes)) if train else (TEST_CLASSES_FROM, bank.n_classes)
        n = max(hi - lo, 0)
        if n_way > n:
            raise ValueError(f"priors.omniglot: {n_way}-way episodes need {n_way} classes; the {'train' if train else 'test'} "
                             f"pool has {n} (bank of {bank.n_classes} classes, num_classes_used={num_classes_used})")
        d.pool_lo, d.pool_n = lo, n
    return d


_KERNEL = "priors.omniglot draws its episodes with the sm_90a Omniglot kernel"


@torch.no_grad()
def sample_episodes(bank, desc, seed=None, device=None):
    """-> x [T, B, S²] fp32, y [T, B] int64, target_y [T, B] int64 on `device` (default: the current CUDA device)."""
    dev = L.compute_device(None, _KERNEL) if device is None else torch.device(device)
    seed = L.draw_seed(seed)
    with L.on_device(dev):
        bank_t, alpha_start = bank.on_device(dev, desc.train)
        x = torch.empty(desc.T, desc.B, desc.S * desc.S, dtype=torch.float32, device=dev)
        y = torch.empty(desc.T, desc.B, dtype=torch.int64, device=dev)
        target_y = torch.empty_like(y)
        L.omniglot_episodes(desc, seed, bank_t, alpha_start, x, y, target_y)
    return x, y, target_y


class DataLoader(PriorDataLoader):
    """The reference's loader (priors/omniglot.py:36-85): `num_steps` batches `((x, y), target_y)` per iteration, sampled on
    the current CUDA device."""

    def __init__(self, num_steps, batch_size, seq_len, num_features, num_outputs, num_classes_used=1200, fuse_x_y=False,
                 train=True, translations=True, jonas_style=False):
        set_locals_in_self(locals())
        assert not fuse_x_y, 'So far don\' support fusing.'
        S, n_way, k_shot = episode_shape(seq_len, num_features, num_outputs)
        self.bank = load_bank(S)
        self.desc = episode_desc(self.bank, batch_size, n_way, k_shot, train=train, jonas_style=jonas_style,
                                 translations=translations, num_classes_used=num_classes_used)

    def __len__(self):
        return self.num_steps

    def __iter__(self):
        L.compute_device(None, _KERNEL)
        return (self._batch() for _ in range(self.num_steps))

    def _batch(self):
        x, y, target_y = sample_episodes(self.bank, self.desc)
        return (x, y), target_y

    @torch.no_grad()
    def validate(self, finetuned_model, eval_pos=-1):
        """Accuracy at row `eval_pos` over `num_steps` test batches of the DEFAULT (not Jonas) mode, as the reference
        does (priors/omniglot.py:74-98).  Leaves the model in eval mode."""
        finetuned_model.eval()
        device = next(iter(finetuned_model.parameters())).device

        if not hasattr(self, 't_dl'):
            self.t_dl = DataLoader(num_steps=self.num_steps, batch_size=self.batch_size, seq_len=self.seq_len,
                                   num_features=self.num_features, num_outputs=self.num_outputs, fuse_x_y=self.fuse_x_y,
                                   train=False)

        ps = []
        ys = []
        for x, y in self.t_dl:
            p = finetuned_model(tuple(e.to(device) for e in x), single_eval_pos=eval_pos)
            ps.append(p)
            ys.append(y)

        ps = torch.cat(ps, 1)
        ys = torch.cat(ys, 1)
        return (ps[eval_pos].argmax(-1) == ys[eval_pos].to(ps.device)).float().mean().cpu()
