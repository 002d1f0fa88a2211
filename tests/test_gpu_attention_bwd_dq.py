"""Tensor-core attention backward, cases aimed at the dQ kernel's software-pipelined key loop and at the per-row statistics
and diagonal keys its producer warps prepare one tile ahead: odd key-block counts with rows >= sep, dropout with several
tiles per CTA (one straddling sep), and bit-identical dqkv across runs."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L
from oracle import error_budget as EB

DH = 128


def _inputs(dev, T, B, H, seed):
    torch.manual_seed(seed)
    E = H * DH
    qkv = (torch.randn(T * B, 3 * E, device=dev) * 1.2).to(torch.bfloat16)
    dout = torch.randn(T * B, E, device=dev).to(torch.bfloat16)
    return qkv, dout


def _check(dqkv, qkv, out, lse, dout, T, B, H, sep, keep=None, drop_scale=1.0):
    assert torch.isfinite(dqkv.float()).all(), "dqkv not fully written"
    f = EB.attention_fwd(qkv, T, B, H, DH, sep, EB.U, keep, drop_scale)
    EB.check_attention_fwd(out, lse, f, EB.C_ATT_OUT, EB.C_ATT_LSE)
    EB.check_attention_bwd(dqkv, EB.attention_bwd(f, dout, out), EB.C_ATT_GRAD)


# 3 and 7 key blocks: odd numbers of blocks through the loop, with query tiles on both sides of sep
@pytest.mark.parametrize("T,B,H,sep", [(300, 2, 2, 150), (600, 3, 2, 420)])
def test_attention_tc_bwd_odd_key_blocks(cuda_device, T, B, H, sep):
    E = H * DH
    qkv, dout = _inputs(cuda_device, T, B, H, T + sep)
    out = torch.empty(T * B, E, device=cuda_device, dtype=torch.bfloat16)
    lse = torch.empty(B * H, T, device=cuda_device)
    L.attention_fwd(qkv, out, lse, T, B, H, DH, sep, use_tc=True)
    dqkv = torch.full_like(qkv, float("nan"))
    delta = torch.empty_like(lse)
    L.attention_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, DH, sep, use_tc=True)
    torch.cuda.synchronize()
    _check(dqkv, qkv, out, lse, dout, T, B, H, sep)


def test_attention_tc_bwd_dropout_several_tiles_per_cta(cuda_device):
    """5 query tiles x 64 (batch, head) pairs: each CTA walks several tiles, and tile 2 straddles sep, so the diagonal
    keep mask and the double-buffered statistics are used across tile boundaries."""
    T, B, H, sep, p = 640, 16, 4, 300, 0.2
    dev, E = cuda_device, H * DH
    thr, seed = L.drop_threshold(p), 515151
    scale = 256.0 / (256 - thr)
    qkv, dout = _inputs(dev, T, B, H, 7)
    out = torch.empty(T * B, E, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B * H, T, device=dev)
    L.attention_fwd(qkv, out, lse, T, B, H, DH, sep, use_tc=True, drop=(seed, thr))
    dqkv = torch.full_like(qkv, float("nan"))
    delta = torch.empty_like(lse)
    L.attention_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, DH, sep, use_tc=True, drop=(seed, thr))
    torch.cuda.synchronize()
    keep = torch.empty(B * H * T, T, device=dev, dtype=torch.uint8)
    L.dropout_keep_mask(keep, seed, thr)
    torch.cuda.synchronize()
    _check(dqkv, qkv, out, lse, dout, T, B, H, sep, keep.reshape(B, H, T, T), scale)


@pytest.mark.parametrize("drop", [False, True])
def test_attention_tc_bwd_deterministic(cuda_device, drop):
    """Two runs on the same inputs write bit-identical dqkv (dq_colsum is left out: its fp32 atomics are unordered)."""
    T, B, H, sep = 1000, 8, 4, 500
    E = H * DH
    qkv, dout = _inputs(cuda_device, T, B, H, 11)
    dr = (99, L.drop_threshold(0.2)) if drop else None
    out = torch.empty(T * B, E, device=cuda_device, dtype=torch.bfloat16)
    lse = torch.empty(B * H, T, device=cuda_device)
    L.attention_fwd(qkv, out, lse, T, B, H, DH, sep, use_tc=True, drop=dr)
    delta = (out.float() * dout.float()).view(T * B, H, DH).sum(-1).contiguous()
    runs = []
    for _ in range(2):
        dqkv = torch.full_like(qkv, float("nan"))
        colsum = torch.zeros(E, device=cuda_device)
        L.attention_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, DH, sep, use_tc=True, drop=dr, dq_colsum=colsum,
                        delta_token_major=True)
        runs.append(dqkv)
    torch.cuda.synchronize()
    assert torch.isfinite(runs[0].float()).all()
    assert torch.equal(runs[0].view(torch.int16), runs[1].view(torch.int16))
