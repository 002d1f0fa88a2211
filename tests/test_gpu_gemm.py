"""wgmma / SIMT GEMM vs the exact fp64 product of the same (bf16-rounded) operands, element by element within the
bounds of oracle/error_budget.py (output rounding, fp32 accumulation over K, the epilogue's own terms)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L
from oracle import error_budget as EB


def _check(name, C, A, B, a_mn=False, b_mn=False, bias=None, aux=None, epilogue="none", fast_gelu=True):
    """C against the exact epilogue(A B^T + bias) of the logical operands (A, B stored MN-major when a_mn / b_mn).
    fast_gelu=False: a SIMT-kernel result (erff GELU, its own accumulation constant)."""
    u = EB.U32 if C.dtype == torch.float32 else EB.U
    ref, bound, _ = EB.gemm(A.t() if a_mn else A, B.t() if b_mn else B, u, EB.C_ACC_TC if fast_gelu else EB.C_ACC_SIMT,
                            bias=bias, aux=aux, epilogue=epilogue, fast_gelu=fast_gelu)
    EB.check(name, C, ref, bound, EB.C_GEMM)


def _operand(rows, cols, mn_major, dtype, dev, ld_pad=0):
    # logical [rows(i), cols(k)]; storage [rows, cols+pad] (K-major) or [cols, rows+pad] (MN-major)
    r8 = lambda n: (n + ld_pad + 7) // 8 * 8 if ld_pad % 8 == 0 else n + ld_pad
    if mn_major:
        buf = torch.randn(cols, r8(rows), device=dev, dtype=torch.float32).to(dtype)
        return buf[:, :rows]
    buf = torch.randn(rows, r8(cols), device=dev, dtype=torch.float32).to(dtype)
    return buf[:, :cols]


CASES = [
    # M, N, K, a_mn, b_mn
    (256, 256, 128, False, False),
    (128, 128, 64, False, False),
    (1000, 1536, 512, False, False),
    (384, 512, 1024, False, False),
    (300, 100, 520, False, False),      # ragged M, N, K tails (TMA zero fill + guarded stores)
    (512, 512, 1536, False, True),      # dgrad: B = W[N_contr, K_out] used MN-major
    (256, 1024, 512, False, True),
    (512, 1536, 2048, True, True),      # wgrad: both MN-major
    (1024, 512, 640, True, True),
    (100, 512, 1000, True, True),
    (256, 384, 256, True, False),
]


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", CASES)
def test_gemm_tc_plain(cuda_device, M, N, K, a_mn, b_mn):
    torch.manual_seed(M + N + K)
    A = _operand(M, K, a_mn, torch.bfloat16, cuda_device, ld_pad=8)
    B = _operand(N, K, b_mn, torch.bfloat16, cuda_device, ld_pad=16)
    C = torch.full((M, (N + 15) // 8 * 8), 7.0, device=cuda_device, dtype=torch.bfloat16)[:, :N]
    L.gemm(A, B, C, a_mn_major=a_mn, b_mn_major=b_mn, M=M, N=N, K=K, use_tc=True)
    torch.cuda.synchronize()
    _check("gemm plain", C, A, B, a_mn, b_mn)


def test_gemm_tc_epilogues(cuda_device):
    torch.manual_seed(0)
    M, N, K = 640, 1024, 512
    A = _operand(M, K, False, torch.bfloat16, cuda_device)
    B = (_operand(N, K, False, torch.bfloat16, cuda_device).float() * 0.05).to(torch.bfloat16)
    bias = torch.randn(N, device=cuda_device)
    aux = torch.randn(M, N, device=cuda_device).to(torch.bfloat16)
    # bias + residual, bf16 out
    C = torch.empty(M, N, device=cuda_device, dtype=torch.bfloat16)
    L.gemm(A, B, C, bias=bias, aux=aux, use_tc=True)
    _check("gemm bias + residual", C, A, B, bias=bias, aux=aux)
    # bias + GELU with saved pre-activation
    C2 = torch.empty_like(C)
    L.gemm(A, B, C, bias=bias, C2=C2, epilogue=L.EPI_GELU, use_tc=True)
    _check("gemm gelu", C, A, B, bias=bias, epilogue="gelu")
    _check("gemm gelu pre-activation", C2, A, B, bias=bias)
    # GELU' epilogue
    L.gemm(A, B, C, aux=aux, epilogue=L.EPI_GELU_BWD, use_tc=True)
    _check("gemm gelu_bwd", C, A, B, aux=aux, epilogue="gelu_bwd")
    # gelu'(pre) in C2 (forward) + plain product with it (backward): the pair that replaces GELU_BWD on the tensor-core path
    L.gemm(A, B, C, bias=bias, C2=C2, epilogue=L.EPI_GELU, c2_gelu_grad=True, use_tc=True)
    _check("gemm gelu (c2 = gelu')", C, A, B, bias=bias, epilogue="gelu")
    _check("gemm c2 gelu'", C2, A, B, bias=bias, epilogue="gelu_grad")
    L.gemm(A, B, C, aux=C2, epilogue=L.EPI_MUL, use_tc=True)
    _check("gemm mul", C, A, B, aux=C2, epilogue="mul")
    # fp32 out
    Cf = torch.empty(M, N, device=cuda_device, dtype=torch.float32)
    L.gemm(A, B, Cf, bias=bias, use_tc=True)
    _check("gemm fp32 out", Cf, A, B, bias=bias)


@pytest.mark.parametrize("M,N,K,b_mn", [(640, 512, 512, True), (300, 256, 192, False), (4096, 512, 512, True)])
def test_gemm_tc_rowdot(cuda_device, M, N, K, b_mn):
    """ROWDOT epilogue: C is the plain product and rowdot[m, g] = sum over column group g of bf16(C[m, n]) * aux[m, n]
    (the attention backward's delta = rowsum(dO * O) per head, produced by the out-projection dgrad)."""
    torch.manual_seed(5)
    width = 128
    A = _operand(M, K, False, torch.bfloat16, cuda_device)
    B = (_operand(N, K, b_mn, torch.bfloat16, cuda_device).float() * 0.05).to(torch.bfloat16)
    aux = torch.randn(M, N, device=cuda_device).to(torch.bfloat16)
    C = torch.empty(M, N, device=cuda_device, dtype=torch.bfloat16)
    rd = torch.zeros(M, N // width, device=cuda_device, dtype=torch.float32)
    L.gemm(A, B, C, b_mn_major=b_mn, aux=aux, epilogue=L.EPI_ROWDOT, rowdot=(rd, width), M=M, N=N, K=K, use_tc=True)
    _check("gemm rowdot C", C, A, B, b_mn=b_mn)                                           # aux is NOT added to C
    exact, bound = EB.rowdot(C, aux, width)                                              # exact w.r.t. the stored C
    EB.check("gemm rowdot", rd, exact, bound, EB.C_ROWDOT)
    with pytest.raises(Exception):                                                       # group width must be a multiple of 128
        L.gemm(A, B, C, b_mn_major=b_mn, aux=aux, epilogue=L.EPI_ROWDOT, rowdot=(rd, 64), M=M, N=N, K=K, use_tc=True)


def test_gemm_tc_splitk_accumulate(cuda_device):
    torch.manual_seed(1)
    M, N, K = 512, 1536, 64 * 200  # wgrad shape: small output, long contraction
    A = _operand(M, K, True, torch.bfloat16, cuda_device)
    B = _operand(N, K, True, torch.bfloat16, cuda_device)
    C = torch.ones(M, N, device=cuda_device, dtype=torch.float32)
    ones = torch.ones_like(C)
    L.gemm(A, B, C, a_mn_major=True, b_mn_major=True, accumulate=True, k_splits=16, use_tc=True)
    _check("gemm split-K wgrad K=12800", C, A, B, True, True, aux=ones)      # the fp32 accumulation term dominates here


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [(100, 70, 33, False, False), (64, 96, 128, False, True),
                                             (50, 40, 300, True, True), (130, 20, 17, True, False)])
def test_gemm_simt(cuda_device, dtype, M, N, K, a_mn, b_mn):
    torch.manual_seed(5)
    A = _operand(M, K, a_mn, dtype, cuda_device, ld_pad=3)
    B = _operand(N, K, b_mn, dtype, cuda_device, ld_pad=1)
    bias = torch.randn(N, device=cuda_device)
    aux = torch.randn(M, N, device=cuda_device).to(dtype)
    C = torch.empty(M, N, device=cuda_device, dtype=dtype)
    C2 = torch.empty(M, N, device=cuda_device, dtype=dtype)
    L.gemm(A, B, C, a_mn_major=a_mn, b_mn_major=b_mn, bias=bias, aux=aux, use_tc=False)
    _check("gemm simt bias + residual", C, A, B, a_mn, b_mn, bias=bias, aux=aux, fast_gelu=False)
    L.gemm(A, B, C, a_mn_major=a_mn, b_mn_major=b_mn, bias=bias, C2=C2, epilogue=L.EPI_GELU, use_tc=False)
    _check("gemm simt gelu", C, A, B, a_mn, b_mn, bias=bias, epilogue="gelu", fast_gelu=False)
    _check("gemm simt gelu pre-activation", C2, A, B, a_mn, b_mn, bias=bias, fast_gelu=False)
    L.gemm(A, B, C, a_mn_major=a_mn, b_mn_major=b_mn, aux=aux, epilogue=L.EPI_GELU_BWD, use_tc=False)
    _check("gemm simt gelu_bwd", C, A, B, a_mn, b_mn, aux=aux, epilogue="gelu_bwd", fast_gelu=False)
    Cf = torch.ones(M, N, device=cuda_device, dtype=torch.float32)
    L.gemm(A, B, Cf, a_mn_major=a_mn, b_mn_major=b_mn, accumulate=True, k_splits=3, use_tc=False)
    _check("gemm simt split-K", Cf, A, B, a_mn, b_mn, aux=torch.ones_like(Cf), fast_gelu=False)


@pytest.mark.parametrize("M,N,K,b_mn", [(40000, 512, 512, False), (40000, 1024, 256, True), (1000, 200, 256, False),
                                        (300, 96, 64, False), (129, 328, 128, True)])
@pytest.mark.parametrize("epi", ["add", "mul"])
def test_gemm_tc_aux_through_staging(cuda_device, M, N, K, b_mn, epi):
    """aux (residual / multiplier) read by the epilogue next to the accumulator: many tiles and k-blocks (ring phases), ragged
    M and N (zero-filled boxes, masked stores), padded aux / C leading dimensions, N narrower and wider than one tile."""
    torch.manual_seed(M + N)
    A = _operand(M, K, False, torch.bfloat16, cuda_device)
    B = (_operand(N, K, b_mn, torch.bfloat16, cuda_device).float() * K ** -0.5).to(torch.bfloat16)
    ldp = (N + 23) // 8 * 8
    aux = torch.randn(M, ldp, device=cuda_device).to(torch.bfloat16)[:, :N]
    C = torch.full((M, ldp + 8), 7.0, device=cuda_device, dtype=torch.bfloat16)[:, :N]
    bias = torch.randn(N, device=cuda_device) if epi == "add" else None
    L.gemm(A, B, C, b_mn_major=b_mn, bias=bias, aux=aux, epilogue=L.EPI_NONE if epi == "add" else L.EPI_MUL,
           M=M, N=N, K=K, use_tc=True)
    if epi == "add":
        _check("gemm aux add", C, A, B, b_mn=b_mn, bias=bias, aux=aux)
    else:
        _check("gemm aux mul", C, A, B, b_mn=b_mn, aux=aux, epilogue="mul")
    assert float(C.untyped_storage().nbytes()) > 0 and torch.all(C.as_strided((M, 8), (ldp + 8, 1), N).float() == 7.0)   # padding untouched
