"""Input encoders with the reference's names (reference encoders.py).  `Linear` feeds the fused embedding kernel;
anything else runs as a regular PyTorch module in front of the CUDA encoder stack.  `Conv` (not in the reference) is
an image encoder on the library's own convolution kernels."""
import math

import torch
import torch.nn as nn

from . import _lib as L
from . import engine

Linear = nn.Linear


class Conv(nn.Module):
    """Image encoder: x [..., S*S] (pixel k = r S + c) -> [..., emsize].  Up to five valid 3x3 convolutions to 64
    channels, each followed by ReLU and applied while the current side is at least 4 (n_conv = min(5, (S - 2) // 2)),
    then the mean over the remaining pixels and Linear(64, emsize).  Runs on the sm_90a kernels of csrc/conv_encoder.cu
    (bf16 NHWC activations on tensor cores, or fp32 FMA in parity mode); convs that are not applied get no gradient, and
    the images themselves none at all."""

    def __init__(self, input_size, emsize):
        super().__init__()
        S = math.isqrt(input_size)
        # L.CONV_MAX_SIDE (112) is the larger of the stroke and Omniglot samplers' largest image sides
        if S * S != input_size or not 4 <= S <= L.CONV_MAX_SIDE:
            raise ValueError(f"encoders.Conv takes square images of side 4 .. {L.CONV_MAX_SIDE}; "
                             f"input_size={input_size} is not one")
        self.convs = nn.ModuleList([nn.Conv2d(1 if i == 0 else 64, 64, 3) for i in range(5)])
        self.linear = nn.Linear(64, emsize)
        self.side = S
        self.n_conv = min(5, (S - 2) // 2)
        self.precision = engine.default_precision()

    def forward(self, x):
        if x.requires_grad:
            raise ValueError("encoders.Conv computes no gradient for its input images; pass a tensor without requires_grad")
        if not x.is_cuda:
            raise RuntimeError(
                "encoders.Conv runs on hand-written sm_90a kernels only; inputs are on "
                f"{x.device}. Move model and data to a CUDA device (there is no CPU fallback).")
        S = self.side
        if x.shape[-1] != S * S:
            raise ValueError(f"encoders.Conv({S * S}, ...) got inputs of {x.shape[-1]} pixels")
        lead = x.shape[:-1]
        params = [p for conv in self.convs[:self.n_conv] for p in (conv.weight, conv.bias)]
        params += [self.linear.weight, self.linear.bias]
        out = engine.ConvEncoderFn.apply(x.reshape(-1, S * S), S, self.precision, torch.is_grad_enabled(), *params)
        return out.reshape(*lead, -1)


class Normalize(nn.Module):
    """(x - mean) / std.  The reference refers to this class without defining it (encoders.py:18); provided so that
    `get_normalized_uniform_encoder` is usable."""

    def __init__(self, mean, std):
        super().__init__()
        self.mean, self.std = mean, std

    def forward(self, x):
        return (x - self.mean) / self.std


def get_normalized_uniform_encoder(encoder_creator):
    """Wrap an encoder fed with U[0,1] features so that it sees zero-mean / unit-std inputs (reference encoders.py:10-18)."""
    return lambda in_dim, out_dim: nn.Sequential(Normalize(.5, math.sqrt(1 / 12)), encoder_creator(in_dim, out_dim))


class CanEmb(nn.Embedding):
    """Per-feature class embedding, concatenated over features (reference encoders.py:22-33)."""

    def __init__(self, num_features, num_embeddings: int, embedding_dim: int, *args, **kwargs):
        assert embedding_dim % num_features == 0
        super().__init__(num_embeddings, embedding_dim // num_features, *args, **kwargs)

    def forward(self, x):
        emb = super().forward(x)
        return emb.view(*emb.shape[:-2], -1)


def get_Canonical(num_classes):
    return lambda num_features, emsize: CanEmb(num_features, num_classes, emsize)
