"""Data parallelism for the PFN step: one process per GPU (torchrun), independent prior draws per rank, ONE NCCL
all-reduce of the flat gradient buffer per optimizer step.  The reference has no distributed
code at all; the semantics implemented here are the ones that reproduce its single-device gradient of the
global-batch mean: grads are summed over ranks, divided by world size, THEN clipped (reference train.py:95-96),
and `single_eval_pos` is identical on every rank for a given step (reference train.py:69 draws one per step).
"""
import os

import torch
import torch.distributed as dist
from torch._utils import _flatten_dense_tensors, _unflatten_dense_tensors


def env_world_size():
    return int(os.environ.get("WORLD_SIZE", "1"))


def init_from_env(device_type="cuda"):
    """Initialise torch.distributed from torchrun's environment (no-op for a single process).  Returns
    (rank, world_size, device)."""
    world = env_world_size()
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if device_type == "cuda" and torch.cuda.is_available():
        torch.cuda.set_device(local_rank)
        device = torch.device("cuda", local_rank)
    else:
        device = torch.device("cpu")
    if world > 1 and not dist.is_initialized():
        backend = "nccl" if device.type == "cuda" else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        if backend == "nccl":
            dist.init_process_group(backend=backend, device_id=device)
        else:
            dist.init_process_group(backend=backend)
    rank = dist.get_rank() if dist.is_initialized() else 0
    return rank, world, device


def world_size():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def rank():
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def broadcast_parameters(module, src=0):
    """Make every rank start from rank `src`'s weights (ranks seed torch differently for distinct prior draws)."""
    if world_size() == 1:
        return
    tensors = [p.data for p in module.parameters()] + [b.data for b in module.buffers() if b.is_floating_point()]
    if not tensors:
        return
    flat = _flatten_dense_tensors(tensors)
    dist.broadcast(flat, src)
    for t, synced in zip(tensors, _unflatten_dense_tensors(flat, tensors)):
        t.copy_(synced)


def allreduce_gradients(params):
    """Average the gradients of `params` over all ranks with a single all-reduce of one flat buffer."""
    w = world_size()
    if w == 1:
        return
    grads = [p.grad for p in params if p.grad is not None]
    if not grads:
        return
    flat = _flatten_dense_tensors(grads)
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    flat.div_(w)
    for g, synced in zip(grads, _unflatten_dense_tensors(flat, grads)):
        g.copy_(synced)


class OverlappedGradReducer:
    """All-reduce of the gradient buckets the engine's backward reports (engine.GRAD_BUCKET_HOOK), overlapped with the rest of
    the backward: every bucket (the decoder's four gradients; the twelve gradients of one encoder layer, last layer first) is
    pre-divided by the world size and all-reduced IN PLACE on NCCL's stream as soon as it is complete in stream order; the
    compute stream only waits for the outstanding collectives right before the gradients are handed to autograd.  Only the
    few remaining parameters (input encoders) go through the plain end-of-step all-reduce.  Sum / world before clipping
    reproduces the single-device gradient of the global-batch mean (reference train.py:92-97)."""

    def __init__(self):
        self.world = world_size()
        self.handles = []
        self.reduced_ptrs = set()
        self.enabled = True

    def install(self, engine_module):
        engine_module.GRAD_BUCKET_HOOK = self.bucket_ready
        engine_module.GRAD_BUCKET_SYNC = self.sync

    def uninstall(self, engine_module):
        engine_module.GRAD_BUCKET_HOOK = None
        engine_module.GRAD_BUCKET_SYNC = None

    def bucket_ready(self, flat):
        if not self.enabled or self.world == 1:
            return
        flat.div_(self.world)
        self.handles.append(dist.all_reduce(flat, op=dist.ReduceOp.SUM, async_op=True))
        self.reduced_ptrs.add((flat.data_ptr(), flat.numel()))

    def sync(self):
        for h in self.handles:
            h.wait()                      # stream-level wait (the host does not block)
        self.handles = []

    def covers(self, grad):
        """True if `grad` lives inside a bucket that was already all-reduced during this backward."""
        p = grad.data_ptr()
        return any(lo <= p < lo + 4 * n for lo, n in self.reduced_ptrs)

    def finish(self, params):
        """End of the backward: all-reduce whatever the buckets did not cover, then forget this step's buckets."""
        self.sync()
        if self.world > 1:
            rest = [p.grad for p in params if p.grad is not None and not self.covers(p.grad)]
            if rest:
                flat = _flatten_dense_tensors(rest)
                dist.all_reduce(flat, op=dist.ReduceOp.SUM)
                flat.div_(self.world)
                for g, synced in zip(rest, _unflatten_dense_tensors(flat, rest)):
                    g.copy_(synced)
        self.reduced_ptrs = set()


def broadcast_object(obj, src=0):
    """Broadcast a small picklable python object (e.g. the epoch's single_eval_pos schedule)."""
    if world_size() == 1:
        return obj
    box = [obj]
    dist.broadcast_object_list(box, src=src)
    return box[0]


def allreduce_mean_scalar(t):
    """Mean over ranks of a scalar / small tensor (loss bookkeeping once per epoch)."""
    if world_size() == 1:
        return t
    t = t.clone()
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t / world_size()
