"""priors.stroke host logic (no GPU): the integer ranges it derives from the reference's keyword fractions, argument
validation before any device work, `use_saved_from`, the loader class and the drop-in registration."""
import sys

import pytest
import torch

from transformerscandobayesianinference_b200.priors import stroke


def test_default_ranges_at_size_28_are_the_references_randint_bounds():
    d = stroke.stroke_desc(28, 5)
    got = (d.strokes_min, d.strokes_max, d.len_min, d.len_max, d.start_min, d.start_max, d.width_min, d.width_max,
           d.offset_min, d.offset_max, d.jitter_min, d.jitter_max)
    assert got == (1, 3, 5, 20, 2, 25, 1, 4, -4, 4, -2, 2)
    assert (d.S, d.C, d.max_iters) == (28, 5, stroke.MAX_ITERS)
    # int() truncation of the scaled fractions, at another size (reference priors/stroke.py:14-16, :49-54)
    d = stroke.stroke_desc(10, 2)
    assert (d.len_min, d.len_max, d.start_min, d.start_max, d.width_min, d.width_max, d.offset_min, d.offset_max,
            d.jitter_min, d.jitter_max) == (int(10 * 5 / 28), int(10 * 20 / 28), 0, 8, 0, 1, -1, 1, 0, 0)


def test_argument_validation_happens_on_the_host():
    with pytest.raises(AssertionError):
        stroke.get_batch(2, 26, num_features=785, num_outputs=5, device='cpu')
    with pytest.raises(AssertionError):
        stroke.get_batch(2, 25, num_features=784, num_outputs=5, only_train_for_last_idx=True, device='cpu')
    with pytest.raises(TypeError, match="unexpected keyword"):
        stroke.get_batch(2, 26, num_features=784, num_outputs=5, min_max_lenght=(0.1, 0.2), device='cpu')
    with pytest.raises(ValueError, match="min_max_len"):
        stroke.get_batch(2, 26, num_features=784, num_outputs=5, min_max_len=(0.5, 0.2), device='cpu')
    with pytest.raises(ValueError, match="image side"):
        stroke.get_batch(2, 26, num_features=200 * 200, num_outputs=5, device='cpu')
    with pytest.raises(ValueError, match="min_max_strokes"):
        stroke.stroke_desc(28, 5, min_max_strokes=(0, 40))


def test_use_saved_from_loads_a_saved_batch(tmp_path):
    d = tmp_path / "len_26_out_5_features_784_bs_3"
    d.mkdir()
    batch = (torch.rand(26, 3, 784), torch.randint(0, 5, (26, 3)), torch.randint(0, 5, (26, 3)))
    torch.save(batch, d / "batch0.pt")
    x, y, t = stroke.get_batch(3, 26, num_features=784, num_outputs=5, use_saved_from=str(tmp_path))
    assert torch.equal(x, batch[0]) and torch.equal(y, batch[1]) and torch.equal(t, batch[2])


def test_normalize_and_loader_class():
    x = torch.arange(6, dtype=torch.float32)
    assert torch.allclose(stroke.normalize(x), (x - x.mean()) / (x.std() + 1e-6))
    assert stroke.DataLoader.num_outputs == 2
    assert stroke.DataLoader.get_batch_method is stroke.get_batch


def test_dropin_registers_priors_stroke():
    import transformerscandobayesianinference_b200 as pfn
    saved = {k: sys.modules.get(k) for k in list(sys.modules) if k.split(".")[0] in pfn._DROPIN_MODULES}
    try:
        pfn.install_dropin()
        assert sys.modules["priors.stroke"] is stroke
    finally:
        for k in [k for k in list(sys.modules) if k.split(".")[0] in pfn._DROPIN_MODULES]:
            del sys.modules[k]
        sys.modules.update({k: v for k, v in saved.items() if v is not None})
