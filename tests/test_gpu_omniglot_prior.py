"""priors.omniglot on the device (csrc/omniglot_prior.cu) against the unmodified reference (reference priors/omniglot.py).

The real Omniglot images are not available to the tests, so they run on a synthetic bank of the reference's shape: 1623
characters x 20 images at 28 x 28 in 30 background and 20 evaluation alphabets of unequal size (`synthetic_bank`).  Every
image is a filled rectangle of grey levels whose top-left pixel is the only black one and whose next eight pixels spell
its index, so each output image decodes (`decode_batch`) to (class, image, rot90 turn, tx, ty) under any turn and shift.

* Structure, for every episode in both modes and both splits: distinct classes from the right pool or alphabet, distinct
  images within a class with the query image outside its class's support, one turn per class (none in Jonas mode),
  consistent labels (class-major support in Jonas mode), target_y, and every image pixel-exact to its turned bank image
  under the NEAREST / fill-0 shift rule (`shift_image`), unshifted unless training with translations.
* Distribution: histograms (`episode_summary`) of 2 000 reference episodes per configuration, recorded by
  `python tools/make_omniglot_golden.py --reference-dir <reference checkout>` in tests/golden/omniglot_prior.pt, against
  the device sampler at fixed seeds (deterministic: the sampler is counter-based); per-bin proportions within 5 standard
  errors of the difference.
* Reproducibility, the empty-image rule, and the notebook's fine-tuning path end to end on the same bank written as a
  PNG tree: `train(...)` with Jonas episodes and translations, `validate`, and `install_dropin()`.
"""
import os
import sys

import numpy as np
import pytest
import torch

from transformerscandobayesianinference_b200 import encoders
from transformerscandobayesianinference_b200.priors import omniglot
from transformerscandobayesianinference_b200.train import Losses, train

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
S, N_WAY, K_SHOT = 28, 5, 5
T = N_WAY * K_SHOT + 1
N_BACKGROUND, N_CLASSES = 964, 1623
CONFIGS = [(jonas, train) for jonas in (False, True) for train in (True, False)]
GOLD_EPISODES = 2000


# ---- shared with tools/make_omniglot_golden.py, which runs the reference loader over exactly this bank -----------------
def alphabet_sizes():
    """30 background alphabets of 964 characters and 20 evaluation alphabets of 659, of unequal sizes (12..54)."""
    def fit(sizes, total):
        sizes = list(sizes)
        while sum(sizes) > total:
            sizes[sizes.index(max(sizes))] -= 1
        return sizes
    return fit([14 + (11 * i) % 41 for i in range(30)], N_BACKGROUND), fit([12 + (17 * i) % 43 for i in range(20)], N_CLASSES - N_BACKGROUND)


def _mix(v):
    v = np.uint64(v)
    with np.errstate(over="ignore"):
        v = (v ^ (v >> np.uint64(33))) * np.uint64(0xFF51AFD7ED558CCD)
        v = (v ^ (v >> np.uint64(33))) * np.uint64(0xC4CEB9FE1A85EC53)
        v ^= v >> np.uint64(33)
    return int(v)


def image_box(idx, size=S):
    """(r0, c0, h, w) of the ink rectangle of image idx = class * 20 + image."""
    h = _mix(idx + 1)
    hh, ww = 3 + h % 10, 3 + (h >> 8) % 10
    return (h >> 16) % (size - hh + 1), (h >> 32) % (size - ww + 1), hh, ww


def image_pattern(idx, hh, ww):
    """[hh, ww] uint8: 0 at the top-left, the 16 bits of idx two per pixel in the next eight pixels (40, 100, 160 or 220),
    then grey filler in 30..229."""
    q = np.arange(hh * ww)
    p = np.array([30 + _mix(idx * 131 + int(k)) % 200 for k in q], dtype=np.int64)
    p[1:9] = 40 + 60 * ((idx >> (2 * (q[1:9] - 1))) & 3)
    p[0] = 0
    return p.reshape(hh, ww).astype(np.uint8)


def synthetic_bank(size=S):
    """(images [1623, 20, size, size] uint8, 255 = background, alphabets [(split, first class, characters)])."""
    bg, ev = alphabet_sizes()
    images = np.full((N_CLASSES, 20, size, size), 255, np.uint8)
    for idx in range(N_CLASSES * 20):
        r0, c0, hh, ww = image_box(idx, size)
        images[idx // 20, idx % 20, r0:r0 + hh, c0:c0 + ww] = image_pattern(idx, hh, ww)
    alphabets, first = [], 0
    for split, sizes in (("background", bg), ("evaluation", ev)):
        for n in sizes:
            alphabets.append((split, first, n))
            first += n
    return images, alphabets


def write_tree(root, images, alphabets):
    """The bank as the reference's extracted tree under root/omniglot/processed (PNG, mode L, source side = S)."""
    from PIL import Image
    for a, (split, first, n) in enumerate(alphabets):
        for c in range(n):
            d = os.path.join(root, "omniglot", "processed", f"images_{split}", f"Alphabet_{a:02d}", f"character{c + 1:02d}")
            os.makedirs(d, exist_ok=True)
            for i in range(20):
                Image.fromarray(images[first + c, i]).save(os.path.join(d, f"{first + c:04d}_{i + 1:02d}.png"))


def shift_image(img, tx, ty):
    """torchvision affine(translate=[tx, ty], NEAREST, fill=0) for integer shifts: out[r][c] = img[r - ty][c - tx]."""
    out = np.zeros_like(img)
    n, m = img.shape
    rs, cs = slice(max(ty, 0), n + min(ty, 0)), slice(max(tx, 0), m + min(tx, 0))
    out[rs, cs] = img[max(-ty, 0):n - max(ty, 0), max(-tx, 0):m - max(tx, 0)]
    return out


def to_float(u8):
    """The reference's 1 - x / 255. in float64, cast to float32."""
    return (1 - u8 / 255.).astype(np.float32)


def _bbox(mask):
    rows, cols = np.nonzero(mask.any(1))[0], np.nonzero(mask.any(0))[0]
    return rows[0], rows[-1], cols[0], cols[-1]


def decode_batch(x, images):
    """x [T, B, S*S] float32 -> int64 [T, B, 9] of (class, image, turn, tx, ty, r0, r1, c0, c1) per image, (r0..c1) being
    the ink box of the turned bank image, checking that each image equals to_float(shift_image(np.rot90(bank image,
    turn), tx, ty)) exactly.  The pixels give the identity; the turn is where the black pixel sits; the shift is the offset
    of the ink box from that of the turned bank image."""
    Tn, Bn, F = x.shape
    size = int(round(F ** 0.5))
    u = np.rint((1 - x.astype(np.float64)) * 255).astype(np.uint8).reshape(Tn, Bn, size, size)
    out = np.zeros((Tn, Bn, 9), np.int64)
    for t in range(Tn):
        for b in range(Bn):
            img = u[t, b]
            r0, r1, c0, c1 = _bbox(img != 255)
            crop = img[r0:r1 + 1, c0:c1 + 1]
            corners = (crop[0, 0], crop[-1, 0], crop[-1, -1], crop[0, -1])      # where turn k puts the top-left pixel
            k = [k for k in range(4) if corners[k] == 0]
            assert len(k) == 1, (t, b)
            k = k[0]
            canon = np.rot90(crop, -k)
            ww = canon.shape[1]
            idx = sum(((int(canon[q // ww, q % ww]) - 40) // 60) << (2 * (q - 1)) for q in range(1, 9))
            rot = np.rot90(images[idx // 20, idx % 20], k)
            box = _bbox(rot != 255)
            tx, ty = c0 - box[2], r0 - box[0]
            expect = to_float(255 - shift_image(255 - rot, tx, ty))
            assert np.array_equal(expect.reshape(-1), x[t, b]), (t, b, idx, k, tx, ty)
            out[t, b] = (idx // 20, idx % 20, k, tx, ty) + tuple(box)
    return out


def episode_summary(dec, y, target_y, images, alphabets, jonas, train, translated, k_shot=K_SHOT, n_way=N_WAY,
                    num_classes_used=1200):
    """Per-episode structural invariants (share of episodes satisfying each) and histograms of one configuration.
    dec [T, B, 9] from decode_batch, y / target_y [T, B] int64 (numpy)."""
    Tn, Bn = y.shape
    size = images.shape[-1]
    split = "background" if train else "evaluation"
    alpha_of = np.zeros(images.shape[0], np.int64)
    pos_in = np.zeros(images.shape[0], np.int64)
    split_alpha = [a for a, (s, _, _) in enumerate(alphabets) if s == split]
    for a, (_, first, n) in enumerate(alphabets):
        alpha_of[first:first + n] = a
        pos_in[first:first + n] = np.arange(n)
    inv = {k: [] for k in ("distinct_classes", "pool", "distinct_images", "query_not_in_support", "rotation", "labels",
                           "class_major", "target", "shift")}
    hist = {"rotation": np.zeros(4, np.int64), "query_label": np.zeros(n_way, np.int64),
            "support_label": np.zeros((Tn - 1, n_way), np.int64), "support_image": np.zeros(20, np.int64),
            "query_image": np.zeros(20, np.int64), "shift": np.zeros((size, size), np.int64),
            "alphabet": np.zeros(len(alphabets), np.int64), "class_decile": np.zeros(17, np.int64)}
    for b in range(Bn):
        cls, img, rot = dec[:, b, 0], dec[:, b, 1], dec[:, b, 2]
        lab = y[:, b]
        by_label = {j: set(cls[lab == j].tolist()) for j in range(n_way)}
        ok_labels = all(len(v) == 1 for v in by_label.values()) and np.array_equal(np.bincount(lab[:-1], minlength=n_way),
                                                                                   np.full(n_way, k_shot))
        inv["labels"].append(ok_labels)
        label_cls = [next(iter(by_label[j])) if len(by_label[j]) == 1 else -1 for j in range(n_way)]
        inv["distinct_classes"].append(len(set(label_cls)) == n_way and -1 not in label_cls)
        if jonas:
            a = alpha_of[label_cls]
            inv["pool"].append(len(set(a.tolist())) == 1 and int(a[0]) in split_alpha
                               and sorted(pos_in[label_cls].tolist()) == list(range(n_way)))
            hist["alphabet"][a[0]] += 1
        else:
            lc = np.array(label_cls)
            inv["pool"].append(bool(((lc < num_classes_used) if train else (lc >= 1200)).all()))
            for c in label_cls:
                hist["class_decile"][c // 100] += 1
        di = qn = rt = True
        for j in range(n_way):
            m = lab[:-1] == j
            sup = img[:-1][m].tolist()
            di &= len(set(sup)) == len(sup)
            if lab[-1] == j:
                qn &= img[-1] not in sup
            rj = rot[lab == j]
            rt &= len(set(rj.tolist())) == 1 and (not jonas or rj[0] == 0)
            hist["rotation"][rj[0]] += 1
        inv["distinct_images"].append(di)
        inv["query_not_in_support"].append(qn)
        inv["rotation"].append(rt)
        inv["class_major"].append(bool(np.array_equal(lab[:-1], np.arange(Tn - 1) // k_shot)))
        inv["target"].append(bool((target_y[:-1, b] == -100).all() and target_y[-1, b] == lab[-1]))
        hist["query_label"][lab[-1]] += 1
        hist["support_label"][np.arange(Tn - 1), lab[:-1]] += 1
        np.add.at(hist["support_image"], img[:-1], 1)
        hist["query_image"][img[-1]] += 1
        if translated:
            sh = True
            for t in range(Tn):
                tx, ty, r0, r1, c0, c1 = dec[t, b, 3:9]
                rx, ry = size - 1 - (c1 - c0), size - 1 - (r1 - r0)          # shifts allowed: rx + 1 and ry + 1
                sh &= -c0 <= tx <= size - 1 - c1 and -r0 <= ty <= size - 1 - r1
                hist["shift"][rx, tx + c0] += 1
                hist["shift"][ry, ty + r0] += 1
            inv["shift"].append(sh)
        else:
            inv["shift"].append(bool((dec[:, b, 3:5] == 0).all()))
    return {"invariants": {k: float(np.mean(v)) for k, v in inv.items()},
            "hist": {k: torch.from_numpy(v) for k, v in hist.items()}, "episodes": Bn}
# ------------------------------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def bank_arrays():
    return synthetic_bank()


@pytest.fixture(scope="module")
def bank(bank_arrays):
    return omniglot.Bank(*bank_arrays)


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(GOLDEN, "omniglot_prior.pt"), weights_only=False)


def _draw(bank, jonas, train, B, seed, translations=True, k_shot=K_SHOT, n_way=N_WAY):
    desc = omniglot.episode_desc(bank, B, n_way, k_shot, train=train, jonas_style=jonas, translations=translations)
    x, y, t = omniglot.sample_episodes(bank, desc, seed=seed, device='cuda:0')
    torch.cuda.synchronize()
    return x.cpu().numpy(), y.cpu().numpy(), t.cpu().numpy()


def _summary(bank, images, alphabets, jonas, train, B, seed, translations=True):
    x, y, t = _draw(bank, jonas, train, B, seed, translations)
    dec = decode_batch(x, images)
    return episode_summary(dec, y, t, images, alphabets, jonas, train, train and translations)


@pytest.mark.parametrize("jonas,train", CONFIGS)
def test_every_episode_has_the_reference_structure(cuda_device, bank, bank_arrays, jonas, train):
    images, alphabets = bank_arrays
    s = _summary(bank, images, alphabets, jonas, train, 1000, 7 + 2 * jonas + train)
    inv = dict(s["invariants"])
    if not jonas:
        assert inv.pop("class_major") < 0.01          # the support is shuffled
    assert all(v == 1.0 for v in inv.values()), inv


def test_no_translation_leaves_images_in_place(cuda_device, bank, bank_arrays):
    images, alphabets = bank_arrays
    for jonas in (False, True):
        s = _summary(bank, images, alphabets, jonas, True, 200, 3, translations=False)
        assert s["invariants"]["shift"] == 1.0 and s["invariants"]["rotation"] == 1.0


def _z_bins(a, b):
    """Largest per-bin |difference of proportions| in pooled standard errors (bins empty in both are skipped)."""
    a, b = a.double().flatten(), b.double().flatten()
    na, nb = a.sum(), b.sum()
    p = (a + b) / (na + nb)
    se = (p * (1 - p) * (1 / na + 1 / nb)).sqrt()
    m = se > 0
    return float(((a / na - b / nb).abs()[m] / se[m]).max()) if m.any() else 0.0


@pytest.mark.parametrize("jonas,train", CONFIGS)
def test_distribution_matches_reference(cuda_device, bank, bank_arrays, gold, jonas, train):
    images, alphabets = bank_arrays
    ref = gold[(jonas, train)]
    ours = _summary(bank, images, alphabets, jonas, train, GOLD_EPISODES, 100 + 2 * jonas + train)
    for k, v in ref["invariants"].items():
        assert ours["invariants"][k] == v or (k == "class_major" and not jonas and v < 0.01), (k, ours["invariants"][k], v)
    for k, h in ref["hist"].items():
        if h.sum() == 0:
            assert ours["hist"][k].sum() == 0, k
            continue
        z = _z_bins(ours["hist"][k], h)
        assert z <= 5, (k, z)


def test_same_seed_same_batch(cuda_device, bank):
    a = _draw(bank, False, True, 64, 5)
    b = _draw(bank, False, True, 64, 5)
    c = _draw(bank, False, True, 64, 6)
    assert all(np.array_equal(u, v) for u, v in zip(a, b))
    assert not np.array_equal(a[0], c[0])
    torch.manual_seed(4)
    d = omniglot.episode_desc(bank, 16, N_WAY, K_SHOT)
    p = omniglot.sample_episodes(bank, d, device='cuda:0')
    torch.manual_seed(4)
    q = omniglot.sample_episodes(bank, d, device='cuda:0')
    assert all(torch.equal(u, v) for u, v in zip(p, q))


def test_layout_odd_side_and_an_image_without_ink(cuda_device):
    # side 13 (S*S not a multiple of 4: scalar stores), 40 classes of which class 3 has one blank image
    rng = np.random.default_rng(0)
    size = 13
    images = np.full((40, 20, size, size), 255, np.uint8)
    images[:, :, 4:8, 5:9] = rng.integers(0, 255, (40, 20, 4, 4), dtype=np.uint8)
    images[1, 7] = 255
    bank = omniglot.Bank(images, [("background", 0, 20), ("evaluation", 20, 20)])
    d = omniglot.episode_desc(bank, 2000, 3, 4, train=True, jonas_style=True)
    x, y, t = omniglot.sample_episodes(bank, d, seed=9, device='cuda:0')
    assert x.shape == (13, 2000, size * size) and x.dtype == torch.float32 and x.is_contiguous()
    assert y.shape == t.shape == (13, 2000) and y.dtype == t.dtype == torch.int64
    x = x.cpu()
    blank = (x == 0).all(-1)
    assert blank.any()                                 # class 1 is among the first 3 characters of alphabet 0
    # every other image: its 4 x 4 ink block shifted within the image, values of the 1 - v / 255 table
    table = torch.from_numpy(to_float(np.arange(256)))
    nz = x[~blank]
    assert torch.isin(nz, table).all()
    assert int((nz != 0).sum(-1).max()) <= 16


def test_host_checks_happen_before_the_launch(bank):
    with pytest.raises(ValueError, match="smallest"):
        omniglot.episode_desc(bank, 4, 13, 1, jonas_style=True, train=False)
    d = omniglot.episode_desc(bank, 4, N_WAY, K_SHOT)
    d.T = 7                                            # the library refuses an inconsistent descriptor itself
    with pytest.raises(RuntimeError, match="T = 7"):
        omniglot.sample_episodes(bank, d, seed=1, device='cuda:0')


@pytest.fixture(scope="module")
def tree(tmp_path_factory, bank_arrays):
    root = tmp_path_factory.mktemp("omniglot_tree")
    write_tree(str(root), *bank_arrays)
    return root


def test_bank_from_the_png_tree(cuda_device, tree, bank_arrays, monkeypatch):
    monkeypatch.chdir(tree)
    b = omniglot.load_bank(S)
    assert np.array_equal(b.images, bank_arrays[0]) and b.alphabets == bank_arrays[1]
    assert omniglot.load_bank(S) is b


def test_notebook_fine_tuning_and_validate(cuda_device, tree, monkeypatch):
    monkeypatch.chdir(tree)
    import transformerscandobayesianinference_b200 as pfn
    saved = {k: sys.modules.get(k) for k in list(sys.modules) if k.split(".")[0] in pfn._DROPIN_MODULES}
    try:
        pfn.install_dropin()
        assert sys.modules["priors.omniglot"] is omniglot
    finally:
        for k in [k for k in list(sys.modules) if k.split(".")[0] in pfn._DROPIN_MODULES]:
            del sys.modules[k]
        sys.modules.update({k: v for k, v in saved.items() if v is not None})
    torch.manual_seed(0)
    kw = {'num_features': S * S, 'fuse_x_y': False, 'num_outputs': N_WAY, 'translations': True, 'jonas_style': True}
    total_loss, _, model = train(omniglot.DataLoader, Losses.ce, encoders.Linear, emsize=256, nhead=2, nhid=512, nlayers=2,
                                 dropout=0.0, epochs=1, steps_per_epoch=3, batch_size=64, bptt=T, lr=1e-4, warmup_epochs=0,
                                 y_encoder_generator=encoders.get_Canonical(N_WAY), extra_prior_kwargs_dict=kw,
                                 single_eval_pos_gen=T - 1, validation_period=1, verbose=False)
    assert np.isfinite(total_loss)
    model = model.to('cuda:0')
    dl = omniglot.DataLoader(num_steps=2, batch_size=32, seq_len=T, **kw)
    torch.manual_seed(11)
    acc = dl.validate(model)
    assert not model.training and dl.t_dl.desc.jonas == 0 and dl.t_dl.desc.train == 0
    torch.manual_seed(11)
    ps, ys = [], []
    with torch.no_grad():
        for (x, y), tgt in dl.t_dl:
            ps.append(model((x, y), single_eval_pos=-1)[-1])
            ys.append(tgt[-1])
    by_hand = (torch.cat(ps).argmax(-1) == torch.cat(ys)).float().mean().cpu()
    assert torch.equal(acc, by_hand), (acc, by_hand)
