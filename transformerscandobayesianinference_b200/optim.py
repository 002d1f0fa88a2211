"""Optimizer step of the training inner loop (reference train.py:94-97) as two kernel launches over all parameters.

    torch.nn.utils.clip_grad_norm_(model.parameters(), 1.)
    optimizer.step()                      # torch.optim.Adam(lr)

`FusedClipAdam` is a `torch.optim.Optimizer` with torch.optim.Adam's constructor arguments, state layout
(`state[p] = {"step", "exp_avg", "exp_avg_sq"}`) and update rule, plus `max_grad_norm` (the clip the reference applies just
before the step).  `step()` hands a device-resident table of (param, grad, exp_avg, exp_avg_sq, bf16 shadow) pointers to
`pfn_adam_step` (csrc/optimizer.cu): one launch for the gradient norm, one for clip + update; the update also rewrites the
bf16 copy of every 2-D weight that the next step's wgmma GEMMs read (engine._cast picks it up), so the per-step cast pass
disappears.  CUDA only: on other devices build torch.optim.Adam (train.py does)."""
import torch

from . import _lib as L

SHADOW_MIN_NUMEL = 1 << 14     # weights below this size are not worth a bf16 shadow (they are not GEMM operands)


class FusedClipAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, max_grad_norm=None,
                 bf16_shadows=True):
        if lr < 0 or eps < 0 or not 0 <= betas[0] < 1 or not 0 <= betas[1] < 1 or weight_decay < 0:
            raise ValueError("FusedClipAdam: invalid hyper-parameters")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self.max_grad_norm = float(max_grad_norm) if max_grad_norm else 0.0
        self.bf16_shadows = bool(bf16_shadows)
        self._tables = {}          # per group: (key of pointers, device table, device chunk_start, n_chunks)
        self._norm_sq = None
        self.last_grad_norm_sq = None

    # ------------------------------------------------------------------ state
    def _init_state(self, p):
        st = self.state[p]
        if "exp_avg" not in st:
            st["step"] = torch.zeros((), dtype=torch.float32)            # torch.optim.Adam keeps the count as a tensor
            st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        return st

    def _shadow(self, p):
        if not (self.bf16_shadows and p.dim() == 2 and p.numel() >= SHADOW_MIN_NUMEL):
            return None
        sh = getattr(p, "_pfn_shadow", None)
        if sh is None or sh[0].shape != p.shape or sh[0].device != p.device:
            sh = [torch.empty(p.shape, device=p.device, dtype=torch.bfloat16), -1]
            p._pfn_shadow = sh
        return sh

    def _table(self, gi, plist):
        chunk = L.adam_chunk_elems()
        entries = []
        for p in plist:
            st = self.state[p]
            sh = self._shadow(p)
            entries.append((p.data_ptr(), p.grad.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(),
                            sh[0].data_ptr() if sh is not None else 0, p.numel()))
        key = tuple(entries)
        cached = self._tables.get(gi)
        if cached is not None and cached[0] == key:
            return cached
        dev = plist[0].device
        host = torch.frombuffer((L.AdamTensor * len(entries))(*entries), dtype=torch.uint8)   # pfn_adam_tensor[n_tensors]
        starts = [0]
        for e in entries:
            starts.append(starts[-1] + (e[5] + chunk - 1) // chunk)
        table = host.pin_memory().to(dev, non_blocking=True)
        chunk_start = torch.tensor(starts, dtype=torch.int32).pin_memory().to(dev, non_blocking=True)
        cached = (key, table, chunk_start, starts[-1])
        self._tables[gi] = cached
        return cached

    # ------------------------------------------------------------------ step
    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        groups = []
        for gi, group in enumerate(self.param_groups):
            plist = [p for p in group["params"] if p.grad is not None]
            if not plist:
                continue
            for p in plist:
                if not (p.is_cuda and p.dtype == torch.float32 and p.grad.dtype == torch.float32 and p.is_contiguous()
                        and p.grad.is_contiguous() and not p.grad.is_sparse):
                    raise RuntimeError("FusedClipAdam: contiguous fp32 CUDA parameters and dense gradients only")
                self._init_state(p)
            groups.append((gi, group, plist))
        if not groups:
            return loss
        if self.max_grad_norm > 0 and len(groups) > 1:
            raise RuntimeError("FusedClipAdam: gradient clipping across several param groups is not implemented")
        dev = groups[0][2][0].device
        if self._norm_sq is None or self._norm_sq.device != dev:
            self._norm_sq = torch.zeros(1, device=dev, dtype=torch.float32)
        for gi, group, plist in groups:
            _, table, chunk_start, n_chunks = self._table(gi, plist)
            st0 = self.state[plist[0]]
            step = int(st0["step"].item()) + 1
            beta1, beta2 = group["betas"]
            L.adam_step(table, chunk_start, len(plist), n_chunks, group["lr"], beta1, beta2, group["eps"],
                        group["weight_decay"], self.max_grad_norm, step, self._norm_sq)
            for p in plist:
                self.state[p]["step"] += 1
                sh = getattr(p, "_pfn_shadow", None)
                if sh is not None:
                    sh[1] = p._version              # the shadow now mirrors this version of the parameter
        self.last_grad_norm_sq = self._norm_sq
        return loss


def cast_weight(w, dtype):
    """The operand copy of a weight in `dtype`: the optimizer's bf16 shadow when it is current, else a fresh cast."""
    sh = getattr(w, "_pfn_shadow", None)
    if sh is not None and dtype == torch.bfloat16 and sh[1] == w._version and sh[0].shape == w.shape and sh[0].device == w.device:
        return sh[0]
    w = w.detach()
    return w.contiguous() if w.dtype == dtype else w.to(dtype).contiguous()
