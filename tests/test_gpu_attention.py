"""Masked attention kernels (fp32-FMA and tensor-core) vs the dense-mask oracle."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L
from oracle import pfn_oracle as O


def _run_fwd(qkv, T, B, H, dh, sep, use_tc):
    dev = qkv.device
    out = torch.empty(T * B, H * dh, device=dev, dtype=qkv.dtype)
    lse = torch.empty(B * H, T, device=dev)
    L.attention_fwd(qkv, out, lse, T, B, H, dh, sep, use_tc=use_tc)
    return out, lse


SIMT_CASES = [(6, 2, 2, 32, 4), (50, 3, 4, 32, 25), (9, 2, 1, 64, 0), (17, 2, 2, 128, 17), (33, 1, 3, 16, 32), (12, 2, 2, 20, 5)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("T,B,H,dh,sep", SIMT_CASES)
def test_attention_simt_fwd_bwd(cuda_device, dtype, T, B, H, dh, sep):
    torch.manual_seed(T * 7 + sep)
    E = H * dh
    qkv = torch.randn(T * B, 3 * E, device=cuda_device).to(dtype)
    out, lse = _run_fwd(qkv, T, B, H, dh, sep, use_tc=False)
    qr = qkv.float().cpu().double().requires_grad_(True)
    ref, ref_lse = O.attention_ref(qr, T, B, H, dh, sep)
    tol = 2e-5 if dtype == torch.float32 else 2e-2
    assert (out.float().cpu().double() - ref).abs().max().item() <= tol * ref.abs().max().item()
    assert (lse.cpu().double() - ref_lse).abs().max().item() <= 1e-4 * (ref_lse.abs().max().item() + 1)
    dout = torch.randn(T * B, E, device=cuda_device).to(dtype)
    (ref * dout.float().cpu().double()).sum().backward()
    dqkv = torch.full_like(qkv, float("nan"))
    delta = torch.empty(B * H, T, device=cuda_device)
    L.attention_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, dh, sep, use_tc=False)
    err = (dqkv.float().cpu().double() - qr.grad).abs().max().item()
    assert err <= (5e-5 if dtype == torch.float32 else 5e-2) * (qr.grad.abs().max().item() + 1e-6), err


# ragged tails (T, sep not multiples of the 64-row tiles / key blocks), sep = 0 and sep = T - 1, and in the last two cases
# more CTAs (B*H*ceil(T/64)) than the GPU holds at once: a tiling error must fail here in seconds, not only in
# tests/test_gpu_fullsize.py
TC_CASES = [(128, 1, 1, 64), (256, 2, 2, 128), (200, 2, 4, 100), (1000, 2, 4, 500), (130, 1, 2, 0), (300, 3, 1, 299),
            (64, 2, 1, 64), (513, 1, 2, 257), (384, 32, 4, 200), (640, 16, 4, 300)]


@pytest.mark.parametrize("T,B,H,sep", TC_CASES)
def test_attention_tc_fwd(cuda_device, T, B, H, sep):
    torch.manual_seed(T + sep)
    dh = 128
    E = H * dh
    qkv = (torch.randn(T * B, 3 * E, device=cuda_device) * 1.5).to(torch.bfloat16)
    out, lse = _run_fwd(qkv, T, B, H, dh, sep, use_tc=True)
    torch.cuda.synchronize()
    ref, ref_lse = O.attention_ref(qkv.float().cpu().double(), T, B, H, dh, sep)
    err = (out.float().cpu().double() - ref).abs().max().item()
    assert err <= 2e-2 * ref.abs().max().item(), f"out err {err}"
    assert (lse.cpu().double() - ref_lse).abs().max().item() <= 2e-3 * (ref_lse.abs().max().item() + 1)


def test_attention_tc_large_scores_rescale(cuda_device):
    # scores spread over a wide range so the lazy-rescale path (running max jumps by > 2^8) is exercised
    torch.manual_seed(11)
    T, B, H, dh, sep = 384, 1, 2, 128, 320
    E = H * dh
    qkv = torch.randn(T * B, 3 * E, device=cuda_device)
    qkv[:, :E] *= 4.0
    qkv[200 * B:260 * B, E:2 * E] *= 6.0   # late key blocks carry much larger scores
    qkv = qkv.to(torch.bfloat16)
    out, lse = _run_fwd(qkv, T, B, H, dh, sep, use_tc=True)
    ref, ref_lse = O.attention_ref(qkv.float().cpu().double(), T, B, H, dh, sep)
    assert (out.float().cpu().double() - ref).abs().max().item() <= 3e-2 * ref.abs().max().item()
    assert (lse.cpu().double() - ref_lse).abs().max().item() <= 2e-3 * (ref_lse.abs().max().item() + 1)


@pytest.mark.parametrize("T,B,H,sep", TC_CASES + [(1000, 1, 2, 1000), (96, 1, 1, 33)])
def test_attention_tc_bwd(cuda_device, T, B, H, sep):
    torch.manual_seed(T * 3 + sep)
    dh = 128
    E = H * dh
    qkv = (torch.randn(T * B, 3 * E, device=cuda_device) * 1.2).to(torch.bfloat16)
    out, lse = _run_fwd(qkv, T, B, H, dh, sep, use_tc=True)
    dout = torch.randn(T * B, E, device=cuda_device).to(torch.bfloat16)
    dqkv = torch.full_like(qkv, float("nan"))
    delta = torch.empty(B * H, T, device=cuda_device)
    L.attention_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, dh, sep, use_tc=True)
    torch.cuda.synchronize()
    qr = qkv.float().cpu().double().requires_grad_(True)
    ref, _ = O.attention_ref(qr, T, B, H, dh, sep)
    (ref * dout.float().cpu().double()).sum().backward()
    got = dqkv.float().cpu().double()
    assert torch.isfinite(got).all(), "dqkv not fully written"
    for name, sl in (("dq", slice(0, E)), ("dk", slice(E, 2 * E)), ("dv", slice(2 * E, 3 * E))):
        want = qr.grad[:, sl]
        err = (got[:, sl] - want).abs().max().item()
        scale_all = qr.grad.abs().max().item()
        assert err <= 3e-2 * want.abs().max().item() + 1e-3 * scale_all, f"{name}: err {err} vs scale {want.abs().max().item()}"
