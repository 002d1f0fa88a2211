"""Paths of the persistent ping-pong wgmma GEMM that the shape cases of test_gpu_gemm.py do not reach: more work units
than CTAs with an odd count per CTA, fp32 output staged over an aux block, split-K with an aux residual in split 0 only,
and a last tile whose second 64-column half lies past N (its aux half is not loaded)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L
from oracle import error_budget as EB


def _check(name, C, A, B, bias=None, aux=None):
    u = EB.U32 if C.dtype == torch.float32 else EB.U
    ref, bound, _ = EB.gemm(A, B, u, EB.C_ACC_TC, bias=bias, aux=aux)
    EB.check(name, C, ref, bound, EB.C_GEMM)


def _rand(rows, cols, dev, scale=1.0):
    return (torch.randn(rows, cols, device=dev) * scale).to(torch.bfloat16)


def test_gemm_tc_units_not_multiple_of_grid(cuda_device):
    """Units = 2 x SMs + 7 tiles: consumer warpgroups of one CTA run different unit counts; residual + bias epilogue."""
    torch.manual_seed(11)
    tiles = 2 * L.num_sms() + 7
    M, N, K = 128 * tiles // 2, 256, 320
    A = _rand(M, K, cuda_device)
    B = _rand(N, K, cuda_device, K ** -0.5)
    bias = torch.randn(N, device=cuda_device)
    aux = _rand(M, N, cuda_device)
    C = torch.empty(M, N, device=cuda_device, dtype=torch.bfloat16)
    L.gemm(A, B, C, bias=bias, aux=aux, use_tc=True)
    _check("gemm units not multiple of grid", C, A, B, bias, aux)


def test_gemm_tc_f32_out_with_aux(cuda_device):
    """fp32 C is staged in two 64-column passes over the slab that held the bf16 aux block."""
    torch.manual_seed(12)
    M, N, K = 1000, 328, 192
    A = _rand(M, K, cuda_device)
    B = _rand(N, K, cuda_device, K ** -0.5)
    bias = torch.randn(N, device=cuda_device)
    aux = _rand(M, N, cuda_device)
    C = torch.full((M, 336), 7.0, device=cuda_device)[:, :N]
    L.gemm(A, B, C, bias=bias, aux=aux, use_tc=True)
    _check("gemm fp32 out with aux", C, A, B, bias, aux)
    assert torch.all(C.as_strided((M, 8), (336, 1), N) == 7.0)          # padding untouched


def test_gemm_tc_splitk_aux_in_first_split(cuda_device):
    """Split-K reduce-add into fp32 with bias and residual: both enter once (split 0), the other splits add products only."""
    torch.manual_seed(13)
    M, N, K = 384, 256, 64 * 40
    A = _rand(M, K, cuda_device)
    B = _rand(N, K, cuda_device, K ** -0.5)
    bias = torch.randn(N, device=cuda_device)
    aux = _rand(M, N, cuda_device)
    C = torch.ones(M, N, device=cuda_device)
    L.gemm(A, B, C, bias=bias, aux=aux, accumulate=True, k_splits=5, use_tc=True)
    _check("gemm split-K aux in first split", C, A, B, bias, aux.float() + 1.0)


def test_gemm_tc_rowdot_ragged_last_group(cuda_device):
    """N = 168: the last tile's second column half is past N, so its staging half keeps a previous tile's data; the row
    dot of the 40-column group must not read it."""
    torch.manual_seed(14)
    M, N, K, width = 2 * 128 * L.num_sms() // 4 + 64, 168, 256, 128
    A = _rand(M, K, cuda_device)
    B = _rand(N, K, cuda_device, 0.05)
    aux = _rand(M, N, cuda_device)
    C = torch.empty(M, N, device=cuda_device, dtype=torch.bfloat16)
    rd = torch.zeros(M, 2, device=cuda_device)
    L.gemm(A, B, C, aux=aux, epilogue=L.EPI_ROWDOT, rowdot=(rd, width), use_tc=True)
    _check("gemm rowdot ragged C", C, A, B)
    exact, bound = EB.rowdot(C, aux, width)
    EB.check("gemm rowdot ragged", rd, exact, bound, EB.C_ROWDOT)
