"""wgmma / SIMT GEMM vs a torch fp32 reference of the same (bf16-rounded) operands."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L


def _ref(A, B, a_mn, b_mn, bias, aux, epi):
    Af = A.float().t() if a_mn else A.float()
    Bf = B.float().t() if b_mn else B.float()
    C = Af @ Bf.t()
    if bias is not None:
        C = C + bias
    pre = C.clone()
    if epi == L.EPI_GELU:
        C = torch.nn.functional.gelu(C)
        if aux is not None:
            C = C + aux.float()
    elif epi == L.EPI_GELU_BWD:
        u = aux.float()
        cdf = 0.5 * (1 + torch.erf(u / 2 ** 0.5))
        pdf = torch.exp(-0.5 * u * u) / (2 * torch.pi) ** 0.5
        C = C * (cdf + u * pdf)
    elif aux is not None:
        C = C + aux.float()
    return C, pre


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
    ref, _ = _ref(A, B, a_mn, b_mn, None, None, L.EPI_NONE)
    torch.cuda.synchronize()
    err = (C.float() - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= 1e-2 * scale + 1e-2, f"max err {err} (scale {scale})"


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
    ref, _ = _ref(A, B, False, False, bias, aux, L.EPI_NONE)
    assert (C.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item()
    # bias + GELU with saved pre-activation
    C2 = torch.empty_like(C)
    L.gemm(A, B, C, bias=bias, C2=C2, epilogue=L.EPI_GELU, use_tc=True)
    ref, pre = _ref(A, B, False, False, bias, None, L.EPI_GELU)
    assert (C.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item()
    assert (C2.float() - pre).abs().max().item() <= 2e-2 * pre.abs().max().item()
    # GELU' epilogue
    L.gemm(A, B, C, aux=aux, epilogue=L.EPI_GELU_BWD, use_tc=True)
    ref, _ = _ref(A, B, False, False, None, aux, L.EPI_GELU_BWD)
    assert (C.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item()
    # gelu'(pre) in C2 (forward) + plain product with it (backward): the pair that replaces GELU_BWD on the tensor-core path
    L.gemm(A, B, C, bias=bias, C2=C2, epilogue=L.EPI_GELU, c2_gelu_grad=True, use_tc=True)
    ref, pre = _ref(A, B, False, False, bias, None, L.EPI_GELU)
    cdf = 0.5 * (1 + torch.erf(pre / 2 ** 0.5))
    gp = cdf + pre * torch.exp(-0.5 * pre * pre) / (2 * torch.pi) ** 0.5
    assert (C.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item()
    assert (C2.float() - gp).abs().max().item() <= 1.5e-2                      # gelu' is O(1); bf16 rounding + approximant
    L.gemm(A, B, C, aux=C2, epilogue=L.EPI_MUL, use_tc=True)
    ref, _ = _ref(A, B, False, False, None, None, L.EPI_NONE)
    ref = ref * C2.float()
    assert (C.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item()
    # fp32 out
    Cf = torch.empty(M, N, device=cuda_device, dtype=torch.float32)
    L.gemm(A, B, Cf, bias=bias, use_tc=True)
    ref, _ = _ref(A, B, False, False, bias, None, L.EPI_NONE)
    assert (Cf - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()


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
    ref, _ = _ref(A, B, False, b_mn, None, None, L.EPI_NONE)
    assert (C.float() - ref).abs().max().item() <= 1e-2 * ref.abs().max().item()       # aux is NOT added to C
    want = (C.float() * aux.float()).view(M, N // width, width).sum(-1)                  # exact w.r.t. the stored C
    assert (rd - want).abs().max().item() <= 1e-4 * want.abs().max().item() + 1e-4
    with pytest.raises(Exception):                                                       # group width must be a multiple of 128
        L.gemm(A, B, C, b_mn_major=b_mn, aux=aux, epilogue=L.EPI_ROWDOT, rowdot=(rd, 64), M=M, N=N, K=K, use_tc=True)


def test_gemm_tc_splitk_accumulate(cuda_device):
    torch.manual_seed(1)
    M, N, K = 512, 1536, 64 * 200  # wgrad shape: small output, long contraction
    A = _operand(M, K, True, torch.bfloat16, cuda_device)
    B = _operand(N, K, True, torch.bfloat16, cuda_device)
    C = torch.ones(M, N, device=cuda_device, dtype=torch.float32)
    L.gemm(A, B, C, a_mn_major=True, b_mn_major=True, accumulate=True, k_splits=16, use_tc=True)
    ref, _ = _ref(A, B, True, True, None, None, L.EPI_NONE)
    ref = ref + 1.0
    assert (C - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()


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
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    L.gemm(A, B, C, a_mn_major=a_mn, b_mn_major=b_mn, bias=bias, aux=aux, use_tc=False)
    ref, _ = _ref(A, B, a_mn, b_mn, bias, aux, L.EPI_NONE)
    assert (C.float() - ref).abs().max().item() <= tol * ref.abs().max().item()
    L.gemm(A, B, C, a_mn_major=a_mn, b_mn_major=b_mn, bias=bias, C2=C2, epilogue=L.EPI_GELU, use_tc=False)
    ref, pre = _ref(A, B, a_mn, b_mn, bias, None, L.EPI_GELU)
    assert (C.float() - ref).abs().max().item() <= tol * ref.abs().max().item()
    assert (C2.float() - pre).abs().max().item() <= tol * pre.abs().max().item()
    L.gemm(A, B, C, a_mn_major=a_mn, b_mn_major=b_mn, aux=aux, epilogue=L.EPI_GELU_BWD, use_tc=False)
    ref, _ = _ref(A, B, a_mn, b_mn, None, aux, L.EPI_GELU_BWD)
    assert (C.float() - ref).abs().max().item() <= tol * ref.abs().max().item()
    Cf = torch.ones(M, N, device=cuda_device, dtype=torch.float32)
    L.gemm(A, B, Cf, a_mn_major=a_mn, b_mn_major=b_mn, accumulate=True, k_splits=3, use_tc=False)
    ref, _ = _ref(A, B, a_mn, b_mn, None, None, L.EPI_NONE)
    assert (Cf - (ref + 1)).abs().max().item() <= max(tol, 1e-5) * (ref.abs().max().item() + 1)


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
    acc = A.float() @ (B.float() if b_mn else B.float().t())
    ref = acc + bias + aux.float() if epi == "add" else acc * aux.float()
    assert (C.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item()
    assert float(C.untyped_storage().nbytes()) > 0 and torch.all(C.as_strided((M, 8), (ldp + 8, 1), N).float() == 7.0)   # padding untouched
