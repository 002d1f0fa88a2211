"""Argument checks of `TransformerModel.encode_context` / `predict` that happen before any device work, so they run on a
CPU model and CPU tensors: unsupported configurations, malformed shapes and contexts that do not fit the model."""
import pytest
import torch

from transformerscandobayesianinference_b200 import encoders, positional_encodings, transformer


def _model(E=64, H=2, L_=2, **kw):
    torch.manual_seed(0)
    return transformer.TransformerModel(encoders.Linear(2, E), 5, E, H, 2 * E, L_, 0.0, y_encoder=encoders.Linear(1, E),
                                        **kw).eval()


def _ctx(n=4, B=3, E=64, nhead=2, nlayers=2, precision=None, device="cpu"):
    precision = precision or _model().precision
    return transformer.TrainingContext(torch.zeros(nlayers, n * B, 2 * E), n, B, E, nhead, nlayers, precision, device)


@pytest.mark.parametrize("kw,reason", [
    (dict(input_normalization=True), "input_normalization"),
    (dict(pos_encoder=positional_encodings.PositionalEncoding(64, 50)), "PositionalEncoding"),
    (dict(pos_encoder=positional_encodings.LearnedPositionalEncoding(64, 50)), "LearnedPositionalEncoding"),
    (dict(pos_encoder=positional_encodings.PairedScrambledPositionalEncodings(64, 50)), "PairedScrambled"),
])
def test_configurations_that_mix_rows_or_positions_are_rejected(kw, reason):
    m = _model(**kw)
    x, y = torch.rand(6, 3, 2), torch.randn(6, 3)
    with pytest.raises(ValueError, match=reason):
        m.encode_context(x, y)
    with pytest.raises(ValueError, match=reason):
        m.predict(_ctx(), x)


def test_training_mode_dropout_is_rejected():
    m = _model()
    m.dropout = 0.1
    m.train()
    with pytest.raises(ValueError, match="dropout"):
        m.encode_context(torch.rand(6, 3, 2), torch.randn(6, 3))
    with pytest.raises(ValueError, match="dropout"):
        m.predict(_ctx(), torch.rand(6, 3, 2))


def test_no_positional_encoding_and_eval_dropout_pass_the_checks():
    """These get as far as the device check (the kernels need CUDA tensors)."""
    m = _model(pos_encoder=positional_encodings.NoPositionalEncoding(64))
    m.dropout = 0.1
    with pytest.raises(RuntimeError, match="CUDA"):
        m.encode_context(torch.rand(6, 3, 2), torch.randn(6, 3))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.predict(_ctx(), torch.rand(6, 3, 2))


@pytest.mark.parametrize("field,value", [("B", 4), ("E", 128), ("nhead", 4), ("nlayers", 3), ("precision", "other"),
                                         ("device", "cuda:0")])
def test_context_that_does_not_fit_is_rejected(field, value):
    ctx = _ctx(**{field: value})
    with pytest.raises(ValueError, match=f"context's {field}"):
        _model().predict(ctx, torch.rand(6, 3, 2))


def test_malformed_arguments_are_rejected():
    m = _model()
    with pytest.raises(ValueError, match="x_train"):
        m.encode_context(torch.rand(6, 3), torch.randn(6, 3))
    with pytest.raises(ValueError, match="y_train"):
        m.encode_context(torch.rand(6, 3, 2), torch.randn(5, 3))
    with pytest.raises(ValueError, match="m >= 1"):
        m.predict(_ctx(), torch.rand(0, 3, 2))
    with pytest.raises(ValueError, match="x_query"):
        m.predict(_ctx(), torch.rand(6, 3))
    with pytest.raises(ValueError, match="TrainingContext"):
        m.predict(object(), torch.rand(6, 3, 2))


def test_timing_script_counts_the_context_attention_work():
    """tools/time_context_inference.py imports without running anything; its FLOPs and bytes follow the shapes."""
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "time_context_inference.py")
    spec = importlib.util.spec_from_file_location("time_context_inference", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    flops, nbytes = mod.attention_work(10, 3, 2)
    E, H, B = mod.E, mod.H, mod.B
    assert flops == 4.0 * 10 * B * H * 4 * (E // H)
    assert nbytes == 2 * (4 * 10 * B * E + 2 * 3 * B * E)
