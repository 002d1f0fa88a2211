"""Drop-in `decoders` (reference decoders.py): the learned-temperature decoder heads, run on the sm_90a engine.

    ScaledDecoder(ninp, nhid, nout)        x -> GELU(linear(x)) -> linear1(.) / (softmax(linear2(.)) . c)
    FixedScaledDecoder(ninp, nhid, nout)   x -> mapper(x) / T.sum()

Parameter names, shapes and construction-time RNG consumption are the reference's, so state dicts load either way and
`torch.manual_seed` gives the same initial weights.  Both heads accept CUDA input of any leading shape; the two GEMMs run
on the tensor-core GEMM and the temperature division in the row kernels of csrc/scaled_head.cu (engine.ScaledDecoderFn,
engine.FixedScaledDecoderFn).  There is no CPU path: a CPU tensor raises RuntimeError.
`TransformerModel(..., decoder=ScaledDecoder)` hands these heads its query rows directly, without the module call.
"""
import random

import torch
from torch import nn

from . import engine

TEMPERATURES = (1., 1.4, 1.7, 2., 5., 10., 20., 40., 80., 160.)     # reference decoders.py:17


def _rows(x, precision):
    if not x.is_cuda:
        raise RuntimeError(
            "decoders run on hand-written sm_90a kernels only; the input is on "
            f"{x.device}. Move the module and data to a CUDA device (there is no CPU fallback).")
    return x.reshape(-1, x.shape[-1]).to(engine.act_dtype(precision))


def _frozen(params, frozen):
    """The head's parameters in the order its engine function takes them, detached when frozen."""
    return [p.detach() if frozen else p for p in params]


class ScaledDecoder(nn.Module):
    """Logits divided by a per-row temperature, the softmax-weighted mean of TEMPERATURES under 10 learned logits.

    Like the reference, every forward makes exactly one `random.random()` draw (the stream `single_eval_pos` sampling
    also uses) and, when it exceeds 0.99, prints `temps.shape, temps[:, :2]`.  `temps` has the leading shape of the
    input: [T - single_eval_pos, B] under `TransformerModel`, which decodes the query rows only, where the reference
    decodes all T rows and prints a [T, B] tensor.  For 2-D input `temps` is 1-D and its first two entries are printed
    (the reference raises IndexError there)."""

    def __init__(self, ninp, nhid, nout):
        super().__init__()
        self.linear = nn.Linear(ninp, nhid)
        self.linear1 = nn.Linear(nhid, nout)
        self.linear2 = nn.Linear(nhid, 10)

    def forward(self, x):
        return self.fused(_rows(x, engine.default_precision()), x.shape[:-1], engine.default_precision())

    def fused(self, h, lead, precision, frozen=False):
        """h [N, ninp] in the activation dtype of `precision` -> logits [*lead, nout] fp32.  frozen: the parameters are
        constants of the call (a backward reaches h only)."""
        params = _frozen((self.linear.weight, self.linear.bias, self.linear1.weight, self.linear1.bias, self.linear2.weight,
                          self.linear2.bias), frozen)
        out, temp = engine.ScaledDecoderFn.apply(h, *params, precision)
        temps = temp.view(lead)
        if random.random() > .99:
            print(temps.shape, temps[:, :2] if temps.dim() >= 2 else temps[:2])
        return out.view(*lead, out.shape[-1])


class FixedScaledDecoder(nn.Module):
    """Logits divided by the sum of a learned 10000-entry parameter T (initially 1)."""

    def __init__(self, ninp, nhid, nout):
        super().__init__()
        self.mapper = nn.Sequential(nn.Linear(ninp, nhid), nn.GELU(), nn.Linear(nhid, nout))
        self.T = nn.Parameter(torch.ones(10000) / 10000)

    def forward(self, x):
        return self.fused(_rows(x, engine.default_precision()), x.shape[:-1], engine.default_precision())

    def fused(self, h, lead, precision, frozen=False):
        """h [N, ninp] in the activation dtype of `precision` -> logits [*lead, nout] fp32.  frozen: the parameters are
        constants of the call (a backward reaches h only)."""
        params = _frozen((self.mapper[0].weight, self.mapper[0].bias, self.mapper[2].weight, self.mapper[2].bias, self.T),
                         frozen)
        out = engine.FixedScaledDecoderFn.apply(h, *params, precision)
        return out.view(*lead, out.shape[-1])
