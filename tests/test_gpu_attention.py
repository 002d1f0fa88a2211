"""Masked attention kernels (fp32-FMA and tensor-core) vs the exact fp64 attention, element by element within the
rounding bounds of oracle/error_budget.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L
from oracle import error_budget as EB


def _run_fwd(qkv, T, B, H, dh, sep, use_tc):
    dev = qkv.device
    out = torch.empty(T * B, H * dh, device=dev, dtype=qkv.dtype)
    lse = torch.empty(B * H, T, device=dev)
    L.attention_fwd(qkv, out, lse, T, B, H, dh, sep, use_tc=use_tc)
    return out, lse


# head dims 160 and 256 run the DPL = 8 instantiation (the stroke notebook's model: emsize 1024, nhead 4); the first of
# them has a ragged sep
SIMT_CASES = [(6, 2, 2, 32, 4), (50, 3, 4, 32, 25), (9, 2, 1, 64, 0), (17, 2, 2, 128, 17), (33, 1, 3, 16, 32), (12, 2, 2, 20, 5),
              (37, 2, 2, 160, 23), (26, 8, 4, 256, 20)]


def _simt_check(qkv, out, lse, dqkv, dout, T, B, H, dh, sep, keep=None, drop_scale=1.0):
    u = EB.U32 if qkv.dtype == torch.float32 else EB.U
    f = EB.attention_fwd(qkv, T, B, H, dh, sep, u, keep, drop_scale)
    EB.check_attention_fwd(out, lse, f, EB.C_ATT_OUT, EB.C_ATT_LSE)
    EB.check_attention_bwd(dqkv, EB.attention_bwd(f, dout, out), EB.C_ATT_GRAD)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("T,B,H,dh,sep", SIMT_CASES)
def test_attention_simt_fwd_bwd(cuda_device, dtype, T, B, H, dh, sep):
    torch.manual_seed(T * 7 + sep)
    E = H * dh
    qkv = torch.randn(T * B, 3 * E, device=cuda_device).to(dtype)
    out, lse = _run_fwd(qkv, T, B, H, dh, sep, use_tc=False)
    dout = torch.randn(T * B, E, device=cuda_device).to(dtype)
    dqkv = torch.full_like(qkv, float("nan"))
    delta = torch.empty(B * H, T, device=cuda_device)
    L.attention_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, dh, sep, use_tc=False)
    torch.cuda.synchronize()
    _simt_check(qkv, out, lse, dqkv, dout, T, B, H, dh, sep)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("T,B,H,dh,sep", [(37, 2, 2, 160, 23), (26, 8, 4, 256, 20)])
def test_attention_simt_dropout(cuda_device, dtype, T, B, H, dh, sep):
    torch.manual_seed(T + dh)
    E = H * dh
    thr, seed = L.drop_threshold(0.2), 777 + dh
    qkv = torch.randn(T * B, 3 * E, device=cuda_device).to(dtype)
    out, lse = torch.empty(T * B, E, device=cuda_device, dtype=dtype), torch.empty(B * H, T, device=cuda_device)
    L.attention_fwd(qkv, out, lse, T, B, H, dh, sep, use_tc=False, drop=(seed, thr))
    dout = torch.randn(T * B, E, device=cuda_device).to(dtype)
    dqkv = torch.full_like(qkv, float("nan"))
    delta = torch.empty(B * H, T, device=cuda_device)
    L.attention_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, dh, sep, use_tc=False, drop=(seed, thr))
    keep = torch.empty(B * H * T, T, device=cuda_device, dtype=torch.uint8)
    L.dropout_keep_mask(keep, seed, thr)
    torch.cuda.synchronize()
    _simt_check(qkv, out, lse, dqkv, dout, T, B, H, dh, sep, keep.reshape(B, H, T, T), 256.0 / (256 - thr))


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
    EB.check_attention_fwd(out, lse, EB.attention_fwd(qkv, T, B, H, dh, sep, EB.U), EB.C_ATT_OUT, EB.C_ATT_LSE)


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
    torch.cuda.synchronize()
    EB.check_attention_fwd(out, lse, EB.attention_fwd(qkv, T, B, H, dh, sep, EB.U), EB.C_ATT_OUT, EB.C_ATT_LSE)


@pytest.mark.parametrize("T,B,H,sep", [(512, 2, 2, 512), (600, 1, 2, 450)])
def test_attention_tc_slowly_rising_max(cuda_device, T, B, H, sep):
    """The running max moves by less than 2 % per key block (oracle.error_budget.rising_max_qkv): every block's O rescale
    is close to 1 but not 1, and the output does not cancel, so a rescale that is skipped or approximated shows."""
    dh = 128
    qkv = EB.rising_max_qkv(T, B, H, dh, torch.Generator().manual_seed(T), device=cuda_device)
    out, lse = _run_fwd(qkv, T, B, H, dh, sep, use_tc=True)
    dout = torch.randn(T * B, H * dh, device=cuda_device).to(torch.bfloat16)
    dqkv = torch.full_like(qkv, float("nan"))
    delta = torch.empty(B * H, T, device=cuda_device)
    L.attention_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, dh, sep, use_tc=True)
    torch.cuda.synchronize()
    f = EB.attention_fwd(qkv, T, B, H, dh, sep, EB.U)
    EB.check_attention_fwd(out, lse, f, EB.C_ATT_OUT, EB.C_ATT_LSE)
    EB.check_attention_bwd(dqkv, EB.attention_bwd(f, dout, out), EB.C_ATT_GRAD)


@pytest.mark.parametrize("T,B,H,sep", TC_CASES + [(1000, 1, 2, 1000), (96, 1, 1, 33), (128, 1, 1, 128), (256, 1, 1, 64),
                                                  (256, 1, 1, 128), (256, 1, 1, 192), (128, 2, 1, 64), (128, 1, 2, 64),
                                                  (200, 1, 1, 100)])
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
    assert torch.isfinite(dqkv.float()).all(), "dqkv not fully written"
    f = EB.attention_fwd(qkv, T, B, H, dh, sep, EB.U)
    EB.check_attention_fwd(out, lse, f, EB.C_ATT_OUT, EB.C_ATT_LSE)
    EB.check_attention_bwd(dqkv, EB.attention_bwd(f, dout, out), EB.C_ATT_GRAD)
