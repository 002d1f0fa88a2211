"""torchrun worker for tests/test_gpu_ragged_training.py::test_two_gpu_ragged_step_gradient: Trainer.step with one
single_eval_pos per dataset of the global batch, through the overlapped bucketed all-reduce, against the single-process
gradient of the global batch's query-row mean."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from transformerscandobayesianinference_b200 import bar_distribution, encoders, parallel, priors, train as T_  # noqa: E402

T, BATCH = 40, 8


def build():
    torch.manual_seed(7)
    crit = bar_distribution.FullSupportBarDistribution(torch.linspace(-4, 4, 21))
    tr = T_.build_trainer(priors.fast_gp.DataLoader, crit, encoders.Linear, emsize=256, nhid=256, nlayers=2, nhead=2,
                          dropout=0.0, epochs=1, steps_per_epoch=2, batch_size=BATCH, bptt=T, lr=0.0, warmup_epochs=0,
                          y_encoder_generator=encoders.Linear, extra_prior_kwargs_dict=dict(num_features=1),
                          single_eval_pos_gen=20)
    tr.model.precision = "fp32"
    with torch.no_grad():
        g = torch.Generator().manual_seed(3)
        for l in tr.model.transformer_encoder.layers:
            l.linear2.weight.copy_(torch.randn(l.linear2.weight.shape, generator=g) * 0.05)
            l.self_attn.out_proj.weight.copy_(torch.randn(l.self_attn.out_proj.weight.shape, generator=g) * 0.05)
    return tr


def main():
    rank, world, dev = parallel.init_from_env("cuda")
    tr = build()
    assert tr.reducer is not None and world == 2
    tr.criterion = tr.criterion.to(dev)
    tr.aggregate_k_gradients = 10 ** 9                      # never step inside .step(); the reduction is finished by hand
    torch.manual_seed(100 + rank)
    x = torch.rand(T, BATCH // world, 1, device=dev); y = torch.randn(T, BATCH // world, device=dev).clamp(-3, 3)
    xs = [torch.zeros_like(x) for _ in range(world)]; ys = [torch.zeros_like(y) for _ in range(world)]
    dist.all_gather(xs, x); dist.all_gather(ys, y)
    X, Y = torch.cat(xs, 1), torch.cat(ys, 1)
    # a ragged batch, and one whose second rank has no query row
    for seps in ([3, 17, 33, 40, 12, 0, 39, 26], [5, 17, 33, 21, 40, 40, 40, 40]):
        tr.optimizer.zero_grad()
        tr.step((x, y), y, seps)
        tr.reducer.finish(tr.params)
        got = [p.grad.clone() for p in tr.params]
        tr.optimizer.zero_grad()
        out = tr.model((X, Y), single_eval_pos=seps)
        s_min = min(seps)
        q = tr.model.query_rows(T, seps).to(dev)
        losses = tr.criterion(out.reshape(-1, 20), Y[s_min:].flatten()).view(T - s_min, BATCH)
        (torch.where(q, losses, 0.).sum() / q.sum()).backward()
        for a, p in zip(got, tr.params):
            assert torch.allclose(a, p.grad, rtol=2e-4, atol=1e-6), \
                f"DP gradient != global-batch gradient for {seps}, shape {tuple(p.shape)}"
    if rank == 0:
        print("DP_RAGGED_WORKER_OK")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
