"""Host-side logic of training with one single_eval_pos per dataset: argument checks of `forward` / `query_rows` /
`utils.per_dataset_sampler`, and the Trainer's masked, globally normalised loss on a fake model and criterion."""
import random

import pytest
import torch
from torch import nn

from transformerscandobayesianinference_b200 import encoders, utils
from transformerscandobayesianinference_b200.train import Trainer
from transformerscandobayesianinference_b200.transformer import TransformerModel


def _model():
    return TransformerModel(encoders.Linear(2, 32), 4, 32, 2, 64, 1, y_encoder=encoders.Linear(1, 32))


@pytest.mark.parametrize("seps,exc,match", [
    ([1, 2], ValueError, "holds 2 values for a batch of 3"),
    ([1, 2, 11], ValueError, r"\[0, 10\]"),
    ([1, -1, 2], ValueError, r"\[0, 10\]"),
    ([1, 2.0, 3], ValueError, "integers"),
    ([1, True, 3], ValueError, "integers"),
    (torch.tensor([1.0, 2.0, 3.0]), ValueError, "integers"),
    (torch.tensor([[1, 2, 3]]), ValueError, "one-dimensional"),
])
def test_forward_rejects_bad_vectors_before_any_kernel(seps, exc, match):
    m = _model()
    x, y = torch.zeros(10, 3, 2), torch.zeros(10, 3)
    with pytest.raises(exc, match=match):
        m((x, y), single_eval_pos=seps)


def test_forward_rejects_a_vector_with_a_mask():
    m = _model()
    x, y = torch.zeros(10, 3, 2), torch.zeros(10, 3)
    with pytest.raises(NotImplementedError, match="src_mask"):
        m((x, y), src_mask=TransformerModel.generate_D_q_matrix(10, 8), single_eval_pos=[2, 3, 4])


def test_query_rows():
    q = TransformerModel.query_rows(6, [2, 4, 6, 3])
    want = torch.tensor([[1, 0, 0, 0], [1, 0, 0, 1], [1, 1, 0, 1], [1, 1, 0, 1]], dtype=torch.bool)
    assert q.dtype == torch.bool and torch.equal(q, want)
    assert torch.equal(TransformerModel.query_rows(6, torch.tensor([2, 4, 6, 3])), want)
    assert TransformerModel.query_rows(6, 4).shape == (2, 1) and TransformerModel.query_rows(6, 4).all()
    assert TransformerModel.query_rows(6, -1).shape == (1, 1)
    with pytest.raises(ValueError, match=r"\[0, 6\]"):
        TransformerModel.query_rows(6, [1, 7])


def test_per_dataset_sampler_draws_the_scalar_stream():
    scalar = utils.get_weighted_single_eval_pos_sampler(20)
    random.seed(4)
    want = [scalar() for _ in range(10)]
    random.seed(4)
    gen = utils.per_dataset_sampler(scalar, 5)
    assert gen() + gen() == want
    for bad in (0, -1, 2.0, True):
        with pytest.raises(ValueError, match="batch_size"):
            utils.per_dataset_sampler(scalar, bad)
    with pytest.raises(ValueError, match="callable"):
        utils.per_dataset_sampler(3, 4)


class _FakeModel(nn.Module):
    """Returns out[r, b] = w * target-independent value for rows t >= min(seps): a differentiable stand-in for forward."""

    def __init__(self, T, B):
        super().__init__()
        self.w = nn.Parameter(torch.ones(()))
        self.vals = torch.arange(T * B, dtype=torch.float32).view(T, B, 1) / 7.0

    def forward(self, data, single_eval_pos):
        s = min(single_eval_pos) if isinstance(single_eval_pos, (list, tuple)) else single_eval_pos
        return self.w * self.vals[s:]

    query_rows = staticmethod(TransformerModel.query_rows)


def _trainer(T, batch, world, rank):
    tr = Trainer.__new__(Trainer)
    tr.device, tr.criterion, tr.n_out = "cpu", nn.MSELoss(reduction="none"), 1
    tr.model = _FakeModel(T, batch // world)
    tr.world, tr.rank, tr.batch_size = world, rank, batch
    tr.reducer, tr.aggregate_k_gradients, tr._micro = None, 1000, 0
    return tr


@pytest.mark.parametrize("world", [1, 2])
def test_trainer_loss_is_the_global_query_row_mean(world):
    T, batch = 6, 4
    seps = [2, 5, 0, 6]
    targets = torch.arange(T * batch, dtype=torch.float32).view(T, batch) % 5
    # the per-row losses of the whole batch, kept on the query rows
    vals = torch.arange(T * (batch // world), dtype=torch.float32).view(T, batch // world) / 7.0
    total, n_query, grads = 0.0, 0, 0.0
    for rank in range(world):
        tr = _trainer(T, batch, world, rank)
        local = slice(rank * batch // world, (rank + 1) * batch // world)
        loss, _ = tr.step((torch.zeros(T, batch // world, 1),) * 2, targets[:, local], seps)
        grads += tr.model.w.grad.item() / world
        total += loss.item() / world
        q = TransformerModel.query_rows(T, seps[local])
        s = min(seps[local])
        n_query += int(q.sum())
        # the exact contribution of this rank to the mean
        grads -= (2 * (vals[s:] - targets[s:, local]) * vals[s:])[q].sum().item() / (sum(T - v for v in seps))
    rows = []
    for b, s in enumerate(seps):
        lb = b % (batch // world)
        rows += [((vals[t, lb] - targets[t, b]) ** 2).item() for t in range(s, T)]
    assert n_query == len(rows) == sum(T - s for s in seps)
    assert total == pytest.approx(sum(rows) / len(rows), rel=1e-6)
    assert grads == pytest.approx(0.0, abs=1e-5)


def test_trainer_rejects_a_step_without_query_rows():
    tr = _trainer(6, 4, 1, 0)
    with pytest.raises(ValueError, match="no query row"):
        tr.step((torch.zeros(6, 4, 1),) * 2, torch.zeros(6, 4), [6, 6, 6, 6])
    with pytest.raises(ValueError, match="holds 3 values for a batch of 4"):
        tr.step((torch.zeros(6, 4, 1),) * 2, torch.zeros(6, 4), [1, 2, 3])
