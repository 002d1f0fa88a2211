"""Host-side helpers under the reference's names (reference utils.py): learning-rate schedules, the `single_eval_pos`
samplers, SeqBN, the OpenAI learning-rate rule and the argparse KEY=VAL action.

Nothing here touches the GPU path.  What matters is that the *streams* agree with the reference: a schedule must return the
same factor for every step, and a sampler must consume python's `random` generator exactly as the reference does (one
`random.choices` call per draw), because `train()` broadcasts nothing but the seed when ranks are expected to agree on
`single_eval_pos`.  `tests/test_host_logic.py` compares both with streams recorded from the unmodified reference."""
import argparse
import math
import random

import torch
from torch import nn
from torch.optim.lr_scheduler import LambdaLR


# ---- learning-rate schedules -----------------------------------------------------------------------------------------
def _warmup_then(decay, num_warmup_steps):
    """LR factor: step / warm-up length while warming up, `decay(step)` (clamped at 0) afterwards."""
    ramp = max(1, num_warmup_steps)

    def factor(step):
        return step / ramp if step < num_warmup_steps else max(0.0, decay(step))
    return factor


def get_cosine_schedule_with_warmup(optimizer, num_warmup_steps, num_training_steps, num_cycles=0.5, last_epoch=-1):
    """Linear warm-up to 1, then 0.5 (1 + cos(2 pi cycles progress))  (reference utils.py:10-22).  `train()` steps the
    schedule once per EPOCH, so with warmup_epochs > 0 the whole first epoch runs at lr 0 (reference train.py:56,134)."""
    span = max(1, num_training_steps - num_warmup_steps)
    cosine = lambda step: 0.5 * (1.0 + math.cos(2.0 * math.pi * num_cycles * ((step - num_warmup_steps) / span)))
    return LambdaLR(optimizer, _warmup_then(cosine, num_warmup_steps), last_epoch)


def get_linear_schedule_with_warmup(optimizer, num_warmup_steps, num_training_steps, last_epoch=-1):
    """Linear warm-up to 1, then a straight line down to 0 at `num_training_steps`  (reference utils.py:25-51)."""
    span = max(1, num_training_steps - num_warmup_steps)
    return LambdaLR(optimizer, _warmup_then(lambda step: (num_training_steps - step) / span, num_warmup_steps), last_epoch)


def get_openai_lr(transformer_model):
    """The OpenAI scaling-law rule lr = 0.003239 - 0.0001395 ln(#parameters)  (reference utils.py:54-56)."""
    return 0.003239 - 0.0001395 * math.log(sum(p.numel() for p in transformer_model.parameters()))


# ---- single_eval_pos samplers -----------------------------------------------------------------------------------------
class _ChoiceSampler:
    """Callable drawing one position per call with ONE `random.choices` call (the reference's stream consumption)."""

    def __init__(self, max_len, weights=None):
        self.population, self.weights = range(max_len), weights

    def __call__(self):
        return random.choices(self.population, self.weights)[0]


def get_weighted_single_eval_pos_sampler(max_len):
    """P(sep = i) proportional to 1 / (max_len - i) over i in [0, max_len): long training sets are favoured so that
    every sequence length contributes about equally many query positions (reference utils.py:59-65)."""
    return _ChoiceSampler(max_len, [1.0 / (max_len - i) for i in range(max_len)])


def get_uniform_single_eval_pos_sampler(max_len):
    """Uniform over [0, max_len)  (reference utils.py:68-73)."""
    return _ChoiceSampler(max_len)


class per_dataset_sampler:
    """Callable drawing one single_eval_pos per dataset: `batch_size` calls of the scalar sampler `sampler` (such as
    get_weighted_single_eval_pos_sampler(k)), returned as a list.  Used as `train(single_eval_pos_gen=...)`, it gives every
    dataset of a step its own training-set size; the draws consume python's `random` as the scalar sampler does."""

    def __init__(self, sampler, batch_size):
        if not callable(sampler):
            raise ValueError(f"per_dataset_sampler: sampler must be callable, got {type(sampler).__name__}")
        if isinstance(batch_size, bool) or not isinstance(batch_size, int) or batch_size < 1:
            raise ValueError(f"per_dataset_sampler: batch_size must be a positive int, got {batch_size!r}")
        self.sampler, self.batch_size = sampler, batch_size

    def __call__(self):
        return [self.sampler() for _ in range(self.batch_size)]


# ---- modules / misc ---------------------------------------------------------------------------------------------------
class SeqBN(nn.Module):
    """BatchNorm1d over all T*B token rows of a [T, B, d_model] tensor (reference utils.py:76-86).  Optional input
    normalisation of `TransformerModel` (off by default); stays a PyTorch module in front of the CUDA stack."""

    def __init__(self, d_model):
        super().__init__()
        self.d_model = d_model
        self.bn = nn.BatchNorm1d(d_model)

    def forward(self, x):
        assert x.shape[-1] == self.d_model
        rows = x.reshape(-1, self.d_model)
        return self.bn(rows).reshape(x.shape)


def set_locals_in_self(locals):
    """`set_locals_in_self(locals())` inside `__init__`: every argument becomes an attribute (reference utils.py:89-93)."""
    target = locals['self']
    for name in locals:
        if name != 'self':
            setattr(target, name, locals[name])


default_device = 'cuda:0' if torch.cuda.is_available() else 'cpu:0'


class StoreDictKeyPair(argparse.Action):
    """`--flag K1=V1 K2=V2 ...` -> {K1: V1, K2: V2}; a value that evaluates as a python expression is stored evaluated,
    anything else as the string it is (reference utils.py:99-113)."""

    def __init__(self, option_strings, dest, nargs=None, **kwargs):
        self._nargs = nargs
        super().__init__(option_strings, dest, nargs=nargs, **kwargs)

    @staticmethod
    def _value(text):
        try:
            return eval(text)
        except NameError:
            return text

    def __call__(self, parser, namespace, values, option_string=None):
        pairs = dict(item.split("=") for item in values)
        parsed = {key: self._value(raw) for key, raw in pairs.items()}
        setattr(namespace, self.dest, parsed)
        print("dict values: {}".format(parsed))
