"""Tensor-core attention forward against the exact fp64 attention (oracle/error_budget.py bounds) on what tests/test_gpu_attention.py does not check directly:
batch-major token order, an output that is a column slice of a wider buffer (the TMA tile store must write exactly the
slice and rows < T), the edges of the persistent tile schedule, and run-to-run determinism."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L
from oracle import error_budget as EB

DH = 128


def _qkv(T, B, H, device):
    torch.manual_seed(T + 7 * B + H)
    return (torch.randn(T * B, 3 * H * DH, device=device) * 1.5).to(torch.bfloat16)


def _check(out, lse, qkv, T, B, H, sep):
    EB.check_attention_fwd(out, lse, EB.attention_fwd(qkv, T, B, H, DH, sep, EB.U), EB.C_ATT_OUT, EB.C_ATT_LSE)


def _fwd(qkv, T, B, H, sep, batch_major=False):
    out = torch.empty(T * B, H * DH, device=qkv.device, dtype=torch.bfloat16)
    lse = torch.empty(B * H, T, device=qkv.device)
    L.attention_fwd(qkv, out, lse, T, B, H, DH, sep, use_tc=True, batch_major=batch_major)
    return out, lse


@pytest.mark.parametrize("T,B,H,sep", [(200, 2, 4, 100), (1000, 2, 4, 500), (130, 1, 2, 0), (300, 3, 1, 299)])
def test_attention_tc_fwd_batch_major(cuda_device, T, B, H, sep):
    qkv = _qkv(T, B, H, cuda_device)
    q_bm = qkv.view(T, B, -1).transpose(0, 1).reshape(T * B, -1).contiguous()
    out_bm, lse = _fwd(q_bm, T, B, H, sep, batch_major=True)
    out = out_bm.view(B, T, -1).transpose(0, 1).reshape(T * B, -1)
    torch.cuda.synchronize()
    _check(out, lse, qkv, T, B, H, sep)


@pytest.mark.parametrize("T,B,H,sep", [(200, 3, 2, 100), (65, 2, 4, 65), (130, 1, 2, 0)])
def test_attention_tc_fwd_strided_out(cuda_device, T, B, H, sep):
    E = H * DH
    qkv = _qkv(T, B, H, cuda_device)
    guard, left, right = 70, 64, 136          # out starts 128 bytes into each row (16-byte aligned), ld_out = E + 200
    buf = torch.full((T * B + guard, left + E + right), float("nan"), device=cuda_device, dtype=torch.bfloat16)
    out = buf[:T * B, left:left + E]
    lse = torch.empty(B * H, T, device=cuda_device)
    L.attention_fwd(qkv, out, lse, T, B, H, DH, sep, use_tc=True)
    torch.cuda.synchronize()
    assert torch.isnan(buf[:, :left]).all() and torch.isnan(buf[:, left + E:]).all(), "columns outside the slice written"
    assert torch.isnan(buf[T * B:]).all(), "guard rows written"
    _check(out, lse, qkv, T, B, H, sep)


# several units per CTA with a count that is not a multiple of the SM count; the cfg-4 shape at small B (the K/V ring
# wraps many times per tile); sep = T (no diagonal rows); a single row; one full tile plus one row with sep = T
@pytest.mark.parametrize("T,B,H,sep", [(1000, 37, 4, 500), (2000, 2, 4, 1000), (384, 3, 2, 384), (1, 1, 1, 0),
                                       (65, 1, 1, 65)])
def test_attention_tc_fwd_schedule_edges(cuda_device, T, B, H, sep):
    qkv = _qkv(T, B, H, cuda_device)
    out, lse = _fwd(qkv, T, B, H, sep)
    torch.cuda.synchronize()
    _check(out, lse, qkv, T, B, H, sep)


def test_attention_tc_fwd_deterministic(cuda_device):
    T, B, H, sep = 1000, 16, 4, 500
    qkv = _qkv(T, B, H, cuda_device)
    out1, lse1 = _fwd(qkv, T, B, H, sep)
    out2, lse2 = _fwd(qkv, T, B, H, sep)
    torch.cuda.synchronize()
    assert torch.equal(out1, out2) and torch.equal(lse1, lse2)
