"""optim.FusedClipAdam (csrc/optimizer.cu) vs torch.nn.utils.clip_grad_norm_ + torch.optim.Adam (reference train.py:55,94-97).

Each step is held element by element to the fp64 restatement of one clip + Adam step (oracle/error_budget.py adam_step)
from the optimizer's own fp32 state before the step, so that rounding does not compound across steps."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L, optim
from oracle import error_budget as EB


def _params(dev, seed):
    g = torch.Generator().manual_seed(seed)
    shapes = [(512, 1536), (100, 1024), (7,), (1024,), (513, 129), (1,), (128, 128)]
    return [torch.nn.Parameter(torch.randn(*s, generator=g).to(dev)) for s in shapes]


class _Checker:
    """Runs opt.step() and checks every tensor against the fp64 step from its state before the step, as it comes;
    `report` prints the worst ratio of each quantity over all steps."""

    def __init__(self, opt, params, lr, wd, max_norm):
        self.opt, self.params, self.lr, self.wd, self.max_norm = opt, params, lr, wd, max_norm
        self.worst = {}
        chunk = L.adam_chunk_elems()
        self.depth = EB.adam_norm_depth(sum((p.numel() + chunk - 1) // chunk for p in params))

    def _check(self, key, got, exact, bound, where):
        r = EB.check(f"adam {key} ({where})", got, exact, bound, EB.C_ADAM, verbose=False)
        self.worst[key] = max(self.worst.get(key, 0.0), r)

    def step(self):
        before = []
        for p in self.params:
            st = self.opt.state.get(p, {})
            m = st["exp_avg"].clone() if "exp_avg" in st else torch.zeros_like(p)
            v = st["exp_avg_sq"].clone() if "exp_avg_sq" in st else torch.zeros_like(p)
            before.append((p.detach().clone(), p.grad.clone(), m, v, int(st["step"].item()) + 1 if "step" in st else 1))
        norm_sq = sum((g.double() ** 2).sum() for _, g, _, _, _ in before).item()
        self.opt.step()
        if self.max_norm:
            got = self.opt.last_grad_norm_sq.double()
            self._check("norm_sq", got, torch.full_like(got, norm_sq), torch.full_like(got, EB.U32 * self.depth * norm_sq),
                        f"step {before[0][4]}")
        for p, (p0, g, m0, v0, step) in zip(self.params, before):
            ex = EB.adam_step(p0, g, m0, v0, step, self.lr, 0.9, 0.999, 1e-8, self.wd, norm_sq, self.max_norm, self.depth)
            st = self.opt.state[p]
            for key, got in (("p", p.detach()), ("m", st["exp_avg"]), ("v", st["exp_avg_sq"])):
                self._check(key, got, ex[key], ex[key + "_bound"], f"step {step}, shape {tuple(p.shape)}")

    def report(self, tag):
        for key, r in self.worst.items():
            print(f"[error-budget] adam {key}{tag}: worst err/bound = {r:.4g} (c = {EB.C_ADAM})")


@pytest.mark.parametrize("max_norm,wd", [(1.0, 0.0), (None, 0.0), (1.0, 0.01)])
def test_fused_clip_adam_matches_torch(cuda_device, max_norm, wd):
    ours = _params(cuda_device, 0)
    opt = optim.FusedClipAdam(ours, lr=3e-3, weight_decay=wd, max_grad_norm=max_norm)
    chk = _Checker(opt, ours, 3e-3, wd, max_norm)
    g = torch.Generator().manual_seed(1)
    for step in range(6):
        scale = 10.0 if step % 2 == 0 else 1e-3          # alternately clipped / not clipped
        for a in ours:
            a.grad = (torch.randn(a.shape, generator=g) * scale).to(cuda_device)
        chk.step()
    chk.report(f" max_norm={max_norm} wd={wd}")
    for a in ours:
        assert float(opt.state[a]["step"]) == 6
    # state_dict round trip into a torch.optim.Adam of the same layout
    topt2 = torch.optim.Adam(_params(cuda_device, 0), lr=3e-3, weight_decay=wd)
    topt2.load_state_dict(opt.state_dict())


def test_adam_flat_gradient_buffer_paths(cuda_device):
    """Gradients handed out as views of one flat fp32 buffer, as the engine does: sizes that are not multiples of 4 put
    the following gradients at offsets that are not 16-byte aligned, so both kernels take their scalar path for them; a
    tensor of several 8192-element chunks with a ragged last one; a vector-path tensor with a scalar tail; 300 steps,
    so that the bias corrections run far from their first-step values.  The bf16 shadow of each 2-D weight must equal
    bf16(p) bit for bit on all three paths."""
    dev = cuda_device
    gen = torch.Generator().manual_seed(7)
    # offsets in floats: 0, 7 (scalar, shadow), 16648 (vector, 3 chunks), 36848 (vector + tail, shadow), 53747 (scalar)
    shapes = [(7,), (129, 129), (200, 101), (129, 131), (5,)]
    ps = [torch.nn.Parameter(torch.randn(*s, generator=gen).to(dev)) for s in shapes]
    sizes = [p.numel() for p in ps]
    flat = torch.empty(sum(sizes), device=dev)
    views, off = [], 0
    for p, n in zip(ps, sizes):
        views.append(flat[off:off + n].view(p.shape))
        off += n
    assert [v.data_ptr() % 16 != 0 for v in views] == [False, True, False, False, True]
    opt = optim.FusedClipAdam(ps, lr=1e-3, weight_decay=0.0, max_grad_norm=1.0)
    chk = _Checker(opt, ps, 1e-3, 0.0, 1.0)
    for step in range(300):
        flat.copy_(torch.randn(flat.numel(), generator=gen).to(dev) * (3.0 if step % 3 == 0 else 1e-3))
        for p, v in zip(ps, views):
            p.grad = v
        chk.step()
        if step % 50 == 0 or step == 299:
            for p in ps:
                sh = getattr(p, "_pfn_shadow", None)
                if p.dim() == 2 and p.numel() >= optim.SHADOW_MIN_NUMEL:
                    assert sh is not None and torch.equal(sh[0], p.detach().to(torch.bfloat16)), (step, p.shape)
    chk.report(" flat buffer, 300 steps")


def test_bf16_shadow_follows_the_parameter(cuda_device):
    ps = _params(cuda_device, 3)
    opt = optim.FusedClipAdam(ps, lr=1e-2, max_grad_norm=1.0)
    w = ps[0]
    assert getattr(w, "_pfn_shadow", None) is None
    c0 = optim.cast_weight(w, torch.bfloat16)
    assert torch.equal(c0, w.detach().to(torch.bfloat16))
    for p in ps:
        p.grad = torch.randn_like(p)
    opt.step()
    sh = optim.cast_weight(w, torch.bfloat16)
    assert sh.data_ptr() == w._pfn_shadow[0].data_ptr()                   # the shadow is used ...
    assert torch.equal(sh, w.detach().to(torch.bfloat16))                 # ... and mirrors the updated weight
    assert getattr(ps[2], "_pfn_shadow", None) is None                    # 1-D parameters get none
    with torch.no_grad():
        w.mul_(2.0)                                                       # an in-place edit invalidates it
    fresh = optim.cast_weight(w, torch.bfloat16)
    assert fresh.data_ptr() != w._pfn_shadow[0].data_ptr() and torch.equal(fresh, w.detach().to(torch.bfloat16))
    for p in ps:
        p.grad = torch.randn_like(p)
    opt.step()                                                            # the next step refreshes it
    assert optim.cast_weight(w, torch.bfloat16).data_ptr() == w._pfn_shadow[0].data_ptr()
    assert torch.equal(w._pfn_shadow[0], w.detach().to(torch.bfloat16))
