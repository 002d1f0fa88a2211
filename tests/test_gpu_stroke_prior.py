"""priors.stroke on the device (csrc/stroke_prior.cu) against the unmodified reference (reference priors/stroke.py).

* Rasteriser and blur, bit for bit: ~22 500 segment sets (regenerated here by `raster_cases`, with the ink fill of
  `raster_fill`) pushed through the oracle hook that runs the sampler's own device functions, against per-image CRC-32
  digests of Pillow's ImageDraw.line mask and GaussianBlur(0.2) outputs recorded in tests/golden/stroke_raster.pt.
* Distribution: summaries (`prior_summary`) of 2 000 reference datasets per mode (tests/golden/stroke_prior.pt) against
  the device sampler at fixed seeds; the sampler is counter-based, so these checks are deterministic.  Thresholds are about
  5 standard errors of the difference, or stated where they are set.
* Layout, normalize_x, determinism (also through the prefetching loader), the rejection cap, and Trainer steps of the
  FewShotOmniglot notebook's setup.
Both fixtures are written by `python tools/make_stroke_golden.py --reference-dir <reference checkout>` (needs PIL).
"""
import math
import os
import random
import zlib

import numpy as np
import pytest
import torch

from transformerscandobayesianinference_b200 import _lib as L, encoders
from transformerscandobayesianinference_b200.priors import stroke
from transformerscandobayesianinference_b200.train import Losses, build_trainer

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
T, C, F = 26, 5, 784
RASTER_SIZES = (28, 3, 10, 32)


# ---- shared with tools/make_stroke_golden.py, which records Pillow's outputs for exactly these inputs -------------------
def raster_cases(S):
    """Deterministic segment sets at image side S: a list of ([(x0, y0, x1, y1), ...], width).  At size 28: every single
    segment with |dx|, |dy| <= 22 from one start point at widths 1-4 (zero-length, horizontal, vertical, diagonal),
    12 000 sampler-like unions of 1-3 strokes over the whole end-point range the prior reaches, and 1 500 sets with end
    points far off every side of the canvas; 300 sets each at sizes 3, 10 and 32."""
    rng = random.Random(2812 + S)
    cases = []
    if S == 28:
        for w in (1, 2, 3, 4):
            for dx in range(-22, 23):
                for dy in range(-22, 23):
                    cases.append(([(13, 14, 13 + dx, 14 + dy)], w))
        for _ in range(12000):
            w, ox, oy, segs = rng.randint(1, 4), rng.randint(-4, 4), rng.randint(-4, 4), []
            for _ in range(rng.randint(1, 3)):
                sx, sy, ln, a = rng.randint(2, 25), rng.randint(2, 25), rng.randint(5, 20), rng.random() * 2 * math.pi
                segs.append((sx + ox, sy + oy, round(sx + ox + math.cos(a) * ln + rng.randint(-2, 2)),
                             round(sy + oy + math.sin(a) * ln + rng.randint(-2, 2))))
            cases.append((segs, w))
        for _ in range(1500):
            cases.append(([tuple(rng.randint(-30, 58) for _ in range(4)) for _ in range(rng.randint(1, 3))], rng.randint(1, 4)))
    else:
        for _ in range(300):
            cases.append(([tuple(rng.randint(-S // 2 - 2, S + S // 2 + 2) for _ in range(4)) for _ in range(rng.randint(1, 3))],
                          rng.randint(1, 4)))
    return cases


def raster_fill(N, S):
    """[N, S*S] uint8 ink fill in U{200..254}: an integer hash of (case, pixel), the same on every platform."""
    i = np.arange(N, dtype=np.uint64)[:, None]
    p = np.arange(S * S, dtype=np.uint64)[None, :]
    with np.errstate(over="ignore"):
        h = i * np.uint64(0x9E3779B97F4A7C15) + p * np.uint64(0xBF58476D1CE4E5B9) + np.uint64(S)
        h ^= h >> np.uint64(31)
        h *= np.uint64(0x94D049BB133111EB)
        h ^= h >> np.uint64(29)
    return (np.uint64(200) + h % np.uint64(55)).astype(np.uint8)


def raster_digests(mask, blur128, blur_fill):
    """Per image: CRC-32 of the 0/1 ink mask, and CRC-32 of the two blurred images (fill 128, then `raster_fill`)."""
    out = np.zeros((mask.shape[0], 2), np.uint32)
    for i in range(mask.shape[0]):
        out[i, 0] = zlib.crc32(np.ascontiguousarray(mask[i], dtype=np.uint8).tobytes())
        out[i, 1] = zlib.crc32(np.ascontiguousarray(blur128[i]).tobytes() + np.ascontiguousarray(blur_fill[i]).tobytes())
    return out


def prior_summary(x, y):
    """Ink-count histogram (pixels > 0.5 per image), per-dataset mean ink and intensity, the mean image, and the mean
    within-class / between-class Pearson correlation of image pairs inside a dataset.  x [T, B, F], y [T, B]."""
    x = x.double()
    T_, B_, F_ = x.shape
    ink = (x > 0.5).sum(-1)                                    # [T, B]
    xc = x - x.mean(-1, keepdim=True)
    xn = (xc / xc.norm(dim=-1, keepdim=True).clamp_min(1e-12)).transpose(0, 1)     # [B, T, F]
    corr = xn @ xn.transpose(1, 2)
    yb = y.transpose(0, 1)
    same = yb.unsqueeze(2) == yb.unsqueeze(1)
    off = ~torch.eye(T_, dtype=torch.bool).unsqueeze(0)
    return {"ink_hist": torch.bincount(ink.flatten(), minlength=F_ + 1).to(torch.int32),
            "ink_ds_mean": ink.double().mean(0).float(), "intensity_ds_mean": x.sum(-1).mean(0).float(),
            "mean_image": x.mean((0, 1)).float(), "corr_within": float(corr[same & off].mean()),
            "corr_between": float(corr[~same].mean())}


def geometry_summary(n_strokes, lengths, starts):
    """Histograms of the class stroke counts, stroke lengths and start coordinates (integer tensors)."""
    return {k: torch.bincount(v.flatten().long(), minlength=m).to(torch.int32)
            for k, v, m in (("n_strokes", n_strokes, 4), ("length", lengths, 21), ("start", starts, 26))}
# ------------------------------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def raster_gold():
    return torch.load(os.path.join(GOLDEN, "stroke_raster.pt"), weights_only=False)


@pytest.fixture(scope="module")
def prior_gold():
    return torch.load(os.path.join(GOLDEN, "stroke_prior.pt"), weights_only=False)


@pytest.mark.parametrize("S", RASTER_SIZES)
def test_raster_and_blur_bit_exact_against_pillow(cuda_device, raster_gold, S):
    cases = raster_cases(S)
    N = len(cases)
    ref = raster_gold["digests"][S].numpy().view(np.uint32)
    assert ref.shape == (N, 2)
    segs = torch.zeros(N, 3, 4, dtype=torch.int32)
    for i, (sg, _) in enumerate(cases):
        segs[i, :len(sg)] = torch.tensor(sg, dtype=torch.int32)
    dev = cuda_device
    nseg = torch.tensor([len(c[0]) for c in cases], dtype=torch.int32, device=dev)
    width = torch.tensor([c[1] for c in cases], dtype=torch.int32, device=dev)
    segs = segs.to(dev)
    mask = torch.empty(N, S * S, dtype=torch.uint8, device=dev)
    b128, bfill, m2 = torch.empty_like(mask), torch.empty_like(mask), torch.empty_like(mask)
    L.stroke_raster(segs, nseg, width, None, mask, b128, S)
    L.stroke_raster(segs, nseg, width, torch.from_numpy(raster_fill(N, S)).to(dev), m2, bfill, S)
    assert torch.equal(mask, m2)
    got = raster_digests(mask.cpu().numpy(), b128.cpu().numpy(), bfill.cpu().numpy())
    for col, name in ((0, "ink mask"), (1, "blurred image")):
        bad = np.nonzero(got[:, col] != ref[:, col])[0]
        assert bad.size == 0, (f"size {S}: {name} differs from Pillow {raster_gold['pillow']} on {bad.size}/{N} images, "
                               f"first {bad[:5].tolist()}: segments {cases[bad[0]][0]} width {cases[bad[0]][1]}")


def _summary_device(seed, last, B=2000):
    torch.manual_seed(seed)
    x, y, _ = stroke.get_batch(B, T, num_features=F, num_outputs=C, only_train_for_last_idx=last, device='cuda:0')
    return prior_summary(x.cpu(), y.cpu())


def _z(a, b):
    a, b = a.double(), b.double()
    return float((a.mean() - b.mean()).abs() / (a.var() / a.numel() + b.var() / b.numel()).sqrt())


def _hist_moments(h):
    h = h.double()
    k = torch.arange(h.numel(), dtype=torch.float64)
    n = h.sum()
    m = (h * k).sum() / n
    return float(m), float(((h * (k - m) ** 2).sum() / (n - 1)).sqrt()), float(n)


def _hist_quantiles(h, qs):
    cdf = h.double().cumsum(0) / h.sum()
    return [int(torch.searchsorted(cdf, torch.tensor([q], dtype=torch.float64))[0]) for q in qs]


def _z_hist(ha, hb):
    (ma, sa, na), (mb, sb, nb) = _hist_moments(ha), _hist_moments(hb)
    return abs(ma - mb) / math.sqrt(sa * sa / na + sb * sb / nb)


@pytest.mark.parametrize("last", [True, False])
def test_distribution_matches_reference(cuda_device, prior_gold, last):
    ref, ours = prior_gold[last], _summary_device(11 + last, last)
    print("ours vs reference: ink", _hist_moments(ours["ink_hist"])[0], _hist_moments(ref["ink_hist"])[0],
          "correlation within", ours["corr_within"], ref["corr_within"], "between", ours["corr_between"], ref["corr_between"])
    # per-dataset means: images of one dataset share its classes, datasets are independent
    for k in ("ink_ds_mean", "intensity_ds_mean"):
        assert _z(ours[k], ref[k]) <= 5, (k, float(ours[k].mean()), float(ref[k].mean()), _z(ours[k], ref[k]))
    # shape of the ink-count distribution: quantiles within 3 pixels, blank images as rare as in the reference
    qs = (0.1, 0.25, 0.5, 0.75, 0.9)
    qa, qb = _hist_quantiles(ours["ink_hist"], qs), _hist_quantiles(ref["ink_hist"], qs)
    assert max(abs(a - b) for a, b in zip(qa, qb)) <= 3, (qa, qb)
    blank_a, blank_b = (float(h[0] / h.sum()) for h in (ours["ink_hist"], ref["ink_hist"]))
    assert blank_a <= 0.005 and blank_b <= 0.005, (blank_a, blank_b)
    # where the ink lies: mean image (per-pixel standard error of the difference is about 0.003)
    d = (ours["mean_image"] - ref["mean_image"]).abs()
    assert float(d.max()) <= 0.03, float(d.max())
    assert float(torch.corrcoef(torch.stack([ours["mean_image"], ref["mean_image"]]))[0, 1]) >= 0.98
    # class structure inside a dataset: images of one class correlate, images of different classes barely
    assert abs(ours["corr_within"] - ref["corr_within"]) <= 0.015, (ours["corr_within"], ref["corr_within"])
    assert abs(ours["corr_between"] - ref["corr_between"]) <= 0.01, (ours["corr_between"], ref["corr_between"])


def test_class_geometry_matches_reference(cuda_device, prior_gold):
    ref = prior_gold["geometry"]
    desc = stroke.stroke_desc(28, C)
    geom, turns, flag = stroke.sample_geometry(2000, desc, 1234, torch.device(cuda_device))
    geom, turns = geom.cpu(), turns.cpu()
    assert int(flag.item()) == 0
    active = geom[..., 3].bool()
    assert not active[..., 1:][~active[..., :1].expand(-1, -1, 2)].any()      # active strokes come first
    ln, st = geom[..., 2][active], geom[..., :2][active].flatten()
    assert ln.min() >= 5 and ln.max() <= 20 and st.min() >= 2 and st.max() <= 25
    ours = geometry_summary(active.sum(-1), ln, st)
    pa, pb = (h.double() / h.sum() for h in (ours["n_strokes"], ref["n_strokes"]))
    assert (pa - pb).abs().max() <= 0.025, (pa.tolist(), pb.tolist())   # s.e. of a difference of proportions near 1/3: 0.0067
    for k in ("length", "start"):
        assert _z_hist(ours[k], ref[k]) <= 5, (k, _hist_moments(ours[k]), _hist_moments(ref[k]))
        assert abs(_hist_moments(ours[k])[1] - _hist_moments(ref[k])[1]) <= 0.2, k
    # every accepted stroke ends inside the canvas (unrounded end point)
    a = 2 * torch.pi * turns[active]
    ex, ey = geom[..., 0][active] + torch.cos(a) * ln, geom[..., 1][active] + torch.sin(a) * ln
    assert float(torch.stack([ex, ey]).min()) >= 0 and float(torch.stack([ex, ey]).max()) <= 27


def test_layout_and_last_index_structure(cuda_device):
    torch.manual_seed(0)
    B = 64
    x, y, t = stroke.get_batch(B, T, num_features=F, num_outputs=C, only_train_for_last_idx=True, device=cuda_device)
    assert x.shape == (T, B, F) and x.dtype == torch.float32 and x.is_cuda and x.is_contiguous()
    assert y.shape == (T, B) and y.dtype == torch.int64 and t.shape == (T, B) and t.dtype == torch.int64
    # ToTensor on the host: uint8 -> float32 divided by 255 (IEEE division; torch's CUDA scalar division would differ)
    xc = x.cpu()
    table = torch.arange(256, dtype=torch.uint8).to(torch.float32).div(255)
    assert torch.equal(table[(xc * 255).round().long()], xc)
    counts = torch.nn.functional.one_hot(y[:-1], C).sum(0)          # [B, C]
    assert (counts == (T - 1) // C).all()
    assert (t[:-1] == -100).all() and torch.equal(t[-1], y[-1]) and y[-1].min() >= 0 and y[-1].max() < C
    # an offset can push a short stroke at the edge off the canvas: the reference leaves about 0.1 % of its images blank
    assert float(((x > 0.5).sum(-1) == 0).double().mean()) <= 0.01
    x2, y2, t2 = stroke.get_batch(B, 10, num_features=100, num_outputs=3, device=cuda_device)
    assert x2.shape == (10, B, 100) and torch.equal(y2, t2) and y2.min() >= 0 and y2.max() < 3 and y2.unique().numel() == 3


def test_normalize_x_matches_torch(cuda_device):
    torch.manual_seed(5)
    x0, y0, _ = stroke.get_batch(32, T, num_features=F, num_outputs=C, only_train_for_last_idx=True, device=cuda_device)
    torch.manual_seed(5)
    x1, y1, _ = stroke.get_batch(32, T, num_features=F, num_outputs=C, only_train_for_last_idx=True, normalize_x=True,
                                 device=cuda_device)
    assert torch.equal(y0, y1)
    ref = (x0 - x0.mean(-1, keepdim=True)) / (x0.std(-1, keepdim=True) + 1e-6)
    torch.testing.assert_close(x1, ref, rtol=1e-5, atol=1e-5)
    assert torch.allclose(stroke.normalize(x0[3, 7]), ref[3, 7], rtol=1e-5, atol=1e-5)


def _loader_batches(monkeypatch, prefetch):
    monkeypatch.setenv("PFN_B200_PREFETCH", "1" if prefetch else "0")
    torch.manual_seed(21)
    dl = stroke.DataLoader(num_steps=3, batch_size=16, seq_len=T, num_features=F, num_outputs=C, only_train_for_last_idx=True,
                           device='cuda:0')
    return [(x.clone(), y.clone(), t.clone()) for (x, y), t in dl]


def test_same_seed_same_batch_and_prefetch_equivalence(cuda_device, monkeypatch):
    torch.manual_seed(3)
    a = stroke.get_batch(16, T, num_features=F, num_outputs=C, device=cuda_device)
    torch.manual_seed(3)
    b = stroke.get_batch(16, T, num_features=F, num_outputs=C, device=cuda_device)
    assert all(torch.equal(u, v) for u, v in zip(a, b))
    c = stroke.get_batch(16, T, num_features=F, num_outputs=C, device=cuda_device)
    assert not torch.equal(a[0], c[0])
    plain, pre = _loader_batches(monkeypatch, False), _loader_batches(monkeypatch, True)
    assert len(plain) == len(pre) == 3
    for p, q in zip(plain, pre):
        assert all(torch.equal(u, v) for u, v in zip(p, q))


def test_rejection_cap_raises(cuda_device, monkeypatch):
    # lengths 42..44 cannot fit in a 28 x 28 canvas from any start point: every stroke hits the cap
    with pytest.raises(stroke.StrokeRejectionError, match=r"min_max_len=\(1.5, 1.6\)"):
        stroke.get_batch(4, T, num_features=F, num_outputs=C, min_max_len=(1.5, 1.6), device=cuda_device)
    monkeypatch.setenv("PFN_B200_PREFETCH", "1")
    dl = stroke.DataLoader(num_steps=2, batch_size=4, seq_len=T, num_features=F, num_outputs=C, min_max_len=(1.5, 1.6),
                           device='cuda:0')
    with pytest.raises(stroke.StrokeRejectionError):
        for _ in dl:
            pass
    x, _, _ = stroke.get_batch(4, T, num_features=F, num_outputs=C, device=cuda_device)     # the device is fine afterwards
    assert torch.isfinite(x).all()


def _notebook_trainer(emsize, nhead, nlayers, B):
    return build_trainer(stroke.DataLoader, Losses.ce, encoders.Linear, emsize=emsize, nhid=2 * emsize, nlayers=nlayers,
                         nhead=nhead, dropout=0.0, epochs=1, steps_per_epoch=3, batch_size=B, bptt=T, lr=1e-4,
                         # no warm-up: a warm-up epoch would hold the learning rate at 0 for the whole epoch
                         warmup_epochs=0, y_encoder_generator=encoders.get_Canonical(C),
                         extra_prior_kwargs_dict={'num_features': F, 'fuse_x_y': False, 'num_outputs': C,
                                                  'only_train_for_last_idx': True},
                         single_eval_pos_gen=T - 1, gpu_device='cuda:0')


# dh = 128 and the notebook's dh = 256.  At least two steps: out_proj and linear2 start at zero (reference
# transformer.py:50-53), so in_proj and linear1 receive no gradient in the first one.
@pytest.mark.parametrize("emsize,nhead,steps", [(256, 2, 3), (512, 2, 2)])
def test_trainer_steps_on_the_notebook_setup(cuda_device, emsize, nhead, steps):
    torch.manual_seed(0)
    tr = _notebook_trainer(emsize, nhead, 2, 64)
    before = [p.detach().clone() for p in tr.model.parameters()]
    done = 0
    for (x, y), targets in tr.dl:
        assert x.shape == (T, 64, F) and y.dtype == torch.int64
        loss, losses = tr.step((x, y), targets, T - 1)
        assert losses.shape == (1, 64) and torch.isfinite(loss).item()
        done += 1
        if done == steps:
            break
    assert done == steps
    changed = [not torch.equal(b, p.detach()) for b, p in zip(before, tr.model.parameters())]
    assert all(changed), sum(changed)
