"""Tensor-core attention backward with the optional inputs the engine uses: the dQ column sums, a precomputed token-major
delta, and batch-major token order."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L
from oracle import error_budget as EB

# ragged T and sep, sep = 0 and sep = T - 1, and more CTAs than the GPU holds at once
CASES = [(200, 2, 4, 100), (1000, 2, 4, 500), (130, 1, 2, 0), (300, 3, 1, 299), (640, 16, 4, 300)]


def _to_batch_major(x, T, B):
    return x.view(T, B, -1).transpose(0, 1).reshape(T * B, -1).contiguous()


def _to_token_major(x, T, B):
    return x.view(B, T, -1).transpose(0, 1).reshape(T * B, -1).contiguous()


@pytest.mark.parametrize("variant", ["dq_colsum", "delta_token_major", "batch_major"])
@pytest.mark.parametrize("T,B,H,sep", CASES)
def test_attention_tc_bwd_inputs(cuda_device, T, B, H, sep, variant):
    torch.manual_seed(T * 3 + sep)
    dh = 128
    E = H * dh
    qkv = (torch.randn(T * B, 3 * E, device=cuda_device) * 1.2).to(torch.bfloat16)
    dout = torch.randn(T * B, E, device=cuda_device).to(torch.bfloat16)
    bm = variant == "batch_major"
    q_in = _to_batch_major(qkv, T, B) if bm else qkv
    d_in = _to_batch_major(dout, T, B) if bm else dout
    out = torch.empty(T * B, E, device=cuda_device, dtype=torch.bfloat16)
    lse = torch.empty(B * H, T, device=cuda_device)
    L.attention_fwd(q_in, out, lse, T, B, H, dh, sep, use_tc=True, batch_major=bm)
    dqkv = torch.full_like(qkv, float("nan"))
    colsum = None
    if variant == "delta_token_major":
        delta = (out.float() * d_in.float()).view(T * B, H, dh).sum(-1).contiguous()
    else:
        delta = torch.empty(B * H, T, device=cuda_device)
    if variant == "dq_colsum":
        colsum = torch.zeros(E, device=cuda_device)
    L.attention_bwd(q_in, out, lse, d_in, dqkv, delta, T, B, H, dh, sep, use_tc=True, batch_major=bm, dq_colsum=colsum,
                    delta_token_major=variant == "delta_token_major")
    torch.cuda.synchronize()
    if bm:
        dqkv = _to_token_major(dqkv, T, B)

    got = dqkv.double()
    assert torch.isfinite(got).all(), "dqkv not fully written"
    out_tm = _to_token_major(out, T, B) if bm else out
    b = EB.attention_bwd(EB.attention_fwd(qkv, T, B, H, dh, sep, EB.U), dout, out_tm)
    EB.check_attention_bwd(got, b, EB.C_ATT_GRAD)
    if colsum is not None:
        cs = colsum.double()
        # the sums are taken over the stored (bf16) dQ: against those, only the order of the fp32 additions differs
        own = got[:, :E].sum(0)
        mag = got[:, :E].abs().sum(0)
        assert ((cs - own).abs() <= 1e-4 * mag + 1e-6).all(), f"colsum vs stored dQ: {(cs - own).abs().max().item()}"
        # against the exact sums: within the sum of the per-element bounds of the column
        EB.check("attention dq_colsum", cs, b["dq"].sum(0), b["dq_bound"].sum(0), EB.C_ATT_GRAD)
