"""Checks of `TransformerModel.encode_context(..., n_train)` that happen before any device work, so they run on a CPU
model and CPU tensors: malformed training-set sizes raise ValueError before anything is launched."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from transformerscandobayesianinference_b200 import _lib as L, encoders, transformer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model(E=64, H=2, L_=2):
    torch.manual_seed(0)
    return transformer.TransformerModel(encoders.Linear(2, E), 5, E, H, 2 * E, L_, 0.0,
                                        y_encoder=encoders.Linear(1, E)).eval()


@pytest.mark.parametrize("n_train,match", [
    ([1, 2], "3 datasets"),
    ([1, 2, 3, 4], "3 datasets"),
    ([1, 2, 7], r"\[0, 6\]"),
    ([-1, 2, 3], r"\[0, 6\]"),
    ([1.0, 2, 3], "integers"),
    ([True, 2, 3], "integers"),
    (torch.tensor([1.0, 2.0, 3.0]), "integers"),
    (torch.tensor([True, False, True]), "integers"),
    (torch.tensor([[1, 2, 3]]), "one-dimensional"),
    (torch.tensor([1, 2, 9]), r"\[0, 6\]"),
    (np.array([1, 2, 3, 4]), "3 datasets"),
])
def test_invalid_sizes_raise_before_any_launch(n_train, match):
    L.reset_launch_count()
    with pytest.raises(ValueError, match=match):
        _model().encode_context(torch.rand(6, 3, 2), torch.randn(6, 3), n_train)
    assert L.launch_count() == 0


@pytest.mark.parametrize("n_train", [[0, 6, 3], (1, 2, 3), np.array([6, 0, 1]), torch.tensor([0, 6, 2], dtype=torch.int16),
                                     torch.tensor([6, 6, 6]), None])
def test_valid_sizes_pass_the_checks(n_train):
    """These get as far as the device check (the kernels need CUDA tensors)."""
    with pytest.raises(RuntimeError, match="CUDA"):
        _model().encode_context(torch.rand(6, 3, 2), torch.randn(6, 3), n_train)


def test_model_checks_come_first():
    m = _model()
    m.dropout = 0.1
    m.train()
    with pytest.raises(ValueError, match="dropout"):
        m.encode_context(torch.rand(6, 3, 2), torch.randn(6, 3), [1, 2, 3])


def test_context_without_sizes_is_uniform():
    ctx = transformer.TrainingContext(torch.zeros(2, 12, 128), 4, 3, 64, 2, 2, "bf16", "cpu")
    assert ctx.n_train is None


def test_timing_script_imports_without_a_device():
    path = os.path.join(ROOT, "tools", "time_ragged_context.py")
    spec = importlib.util.spec_from_file_location("time_ragged_context", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert mod.BNN_SIZES == list(range(2, 93, 5)) and len(mod.BNN_SIZES) == 19
    assert [s["E"] for s in mod.SHAPES.values()] == [256, 512]
