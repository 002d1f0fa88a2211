"""Training with one single_eval_pos per dataset under data parallelism on CPU (world 2, gloo): the values drawn on rank 0
reach every rank, each rank takes its slice, the all-reduced gradient of the masked loss is the gradient of the global
batch's query-row mean (also when one rank's slice has no query row), and the positional losses are the global
per-dataset means.  The model is a differentiable stand-in; the kernels are covered by tests/test_gpu_ragged_training.py."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from torch import nn

T, BATCH = 6, 4


class _Model(nn.Module):
    """out[r, b] = w * x[s + r, b] for the rows from s = min(single_eval_pos)."""

    def __init__(self):
        super().__init__()
        self.w = nn.Parameter(torch.tensor(0.5))

    def forward(self, data, single_eval_pos):
        s = min(single_eval_pos) if isinstance(single_eval_pos, (list, tuple)) else single_eval_pos
        return (self.w * data[0][s:]).unsqueeze(-1)


def _trainer(world, rank, gen):
    from transformerscandobayesianinference_b200.train import Trainer
    tr = Trainer.__new__(Trainer)
    tr.device, tr.criterion, tr.n_out = "cpu", nn.MSELoss(reduction="none"), 1
    tr.model = _Model()
    tr.params = list(tr.model.parameters())
    tr.optimizer = torch.optim.SGD(tr.params, lr=0.0)
    tr.world, tr.rank, tr.batch_size = world, rank, BATCH
    tr.reducer, tr.aggregate_k_gradients, tr._micro = None, 10 ** 9, 0
    tr.single_eval_pos_gen, tr.bptt, tr.steps_per_epoch = gen, T, 2
    return tr


def _data(step):
    g = torch.Generator().manual_seed(step)
    return torch.randn(T, BATCH, generator=g), torch.randn(T, BATCH, generator=g)


def _global_reference(seps, x, y):
    """Gradient of the mean over the query rows of the whole batch, and each dataset's mean query-row loss."""
    w = torch.tensor(0.5, requires_grad=True)
    q = torch.arange(T).unsqueeze(1) >= torch.tensor(seps).unsqueeze(0)
    losses = (w * x - y) ** 2
    losses[q].mean().backward()
    per = [losses[:, b][q[:, b]].mean().item() for b in range(BATCH) if seps[b] < T]
    return w.grad.item(), per


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import random
    from transformerscandobayesianinference_b200 import parallel, utils
    parallel.init_from_env(device_type="cpu")
    local = BATCH // world
    sl = slice(rank * local, (rank + 1) * local)
    # the step: a ragged batch, and one whose second half has no query row
    for step, seps in enumerate(([1, 4, 0, 5], [2, 3, T, T])):
        x, y = _data(step)
        tr = _trainer(world, rank, None)
        tr.step((x[:, sl], y[:, sl]), y[:, sl], seps)
        parallel.allreduce_gradients(tr.params)
        want, _ = _global_reference(seps, x, y)
        assert tr.model.w.grad.item() == pytest.approx(want, rel=1e-5), (rank, seps)
    # an epoch: the values drawn on rank 0 are the ones every rank uses, the positional losses are the global means
    random.seed(11 + rank)
    tr = _trainer(world, rank, utils.per_dataset_sampler(utils.get_uniform_single_eval_pos_sampler(T), BATCH))
    tr.aggregate_k_gradients = 2
    tr.dl = [((_data(10 + i)[0][:, sl], _data(10 + i)[1][:, sl]), _data(10 + i)[1][:, sl]) for i in range(2)]
    drawn = []
    orig = tr.draw_single_eval_positions
    tr.draw_single_eval_positions = lambda n: drawn.extend(orig(n)) or drawn
    _, pos_losses, *_ = tr.train_epoch()
    gathered = [None] * world
    dist.all_gather_object(gathered, drawn)
    assert gathered[0] == gathered[1] and len(drawn) == 2 and all(len(v) == BATCH for v in drawn)
    sums, counts = [0.0] * T, [0] * T
    for i, seps in enumerate(drawn):
        x, y = _data(10 + i)
        for s, v in zip([s for s in seps if s < T], _global_reference(seps, x, y)[1]):
            sums[s] += v
            counts[s] += 1
    for s in range(T):
        if counts[s]:
            assert pos_losses[s] == pytest.approx(sums[s] / counts[s], rel=1e-5), s
    ret[rank] = True
    dist.destroy_process_group()


def test_gloo_world2_ragged_training():
    world = 2
    port = 29300 + os.getpid() % 250
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
    assert dict(ret) == {0: True, 1: True}
