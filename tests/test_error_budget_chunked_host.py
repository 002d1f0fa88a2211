"""The chunked forms of the error-budget helpers (oracle/error_budget.py) against their whole-tensor forms: a full-size
step's weight gradients, LayerNorm and embedding column sums contract over 512 000 tokens, where an fp64 copy of one
operand is several GB, so the full-size checks take the exact values and bounds a block of tokens at a time.  Chunked
and whole agree to fp64 rounding, also when the block does not divide the token count."""
import pytest
import torch

from oracle import error_budget as EB

NUM_SMS = 132


def _close(a, b):
    a, b = a.double(), b.double()
    assert a.shape == b.shape
    assert torch.allclose(a, b, rtol=1e-12, atol=1e-300), (a - b).abs().max().item()


def _bf16(*shape, g, scale=1.0, offset=0.0):
    return (torch.randn(*shape, generator=g, dtype=torch.float64) * scale + offset).to(torch.bfloat16)


@pytest.mark.parametrize("block", [64, 100, 333, 1000, 4096])
def test_wgrad_gemm_chunked_matches_whole(block):
    """The wgrad form: dW [N, K] = dY^T X over the tokens, both operands read MN-major (logical dY^T [N, tokens])."""
    g = torch.Generator().manual_seed(21)
    tokens, N, K = 1000, 48, 40
    dy, x = _bf16(tokens, N, g=g), _bf16(tokens, K, g=g, offset=0.5)       # x with a mean: one-signed products
    init = torch.randn(N, K, generator=g, dtype=torch.float32)
    ex, bd, _ = EB.gemm(dy.t(), x.t(), EB.U32, EB.C_ACC_WGRAD, aux=init)
    exc, bdc, _ = EB.gemm(dy.t(), x.t(), EB.U32, EB.C_ACC_WGRAD, aux=init, block_k=block)
    _close(exc, ex)
    _close(bdc, bd)


def test_gemm_unchunked_is_unchanged():
    """block_k covering the whole contraction gives the whole-tensor result bit for bit."""
    g = torch.Generator().manual_seed(22)
    A, B = _bf16(16, 300, g=g), _bf16(24, 300, g=g)
    ex, bd, _ = EB.gemm(A, B, EB.U32, EB.C_ACC_TC)
    exc, bdc, _ = EB.gemm(A, B, EB.U32, EB.C_ACC_TC, block_k=300)
    assert torch.equal(ex, exc) and torch.equal(bd, bdc)


@pytest.mark.parametrize("block", [7, 64, 250, 999])
def test_layernorm_bwd_chunked_matches_whole(block):
    g = torch.Generator().manual_seed(23)
    rows, E = 999, 64
    z = _bf16(rows, E, g=g, scale=2.0, offset=0.3)
    dh = _bf16(rows, E, g=g)
    gamma = 1.0 + 0.1 * torch.randn(E, generator=g)
    zd = z.double()
    mean = zd.mean(-1).float()
    rstd = (1.0 / torch.sqrt(((zd - zd.mean(-1, keepdim=True)) ** 2).mean(-1) + 1e-5)).float()
    init = [torch.randn(E, generator=g) for _ in range(3)]
    depth = EB.ln_bwd_colsum_depth(rows, E, 2, True, NUM_SMS)
    whole = EB.layernorm_bwd(dh, z, gamma, mean, rstd, EB.U, depth, init)
    part = EB.layernorm_bwd(dh, z, gamma, mean, rstd, EB.U, depth, init, block_rows=block)
    assert "dz" not in part and "dz_bound" not in part
    for k in ("dgamma", "dgamma_bound", "dbeta", "dbeta_bound", "colsum", "colsum_bound", "dz_bound_sum"):
        _close(part[k], whole[k])
    _close(whole["dz_bound_sum"], whole["dz_bound"].sum(0))


@pytest.mark.parametrize("block", [5, 512, 700, 3000])
def test_embed_bwd_chunked_matches_whole(block):
    """The train rows (the first sep*B) straddle block boundaries."""
    g = torch.Generator().manual_seed(24)
    rows, F, E, train = 1300, 3, 32, 650
    dout = _bf16(rows, E, g=g)
    x, y = torch.rand(rows, F, generator=g), torch.randn(rows, generator=g)
    depth = EB.embed_bwd_depth(rows)
    whole = EB.embed_bwd(dout, x, y, train, depth)
    part = EB.embed_bwd(dout, x, y, train, depth, block_rows=block)
    for k in ("dWx", "dbx", "dwy", "dby"):
        _close(part[k][0], whole[k][0])
        _close(part[k][1], whole[k][1])


def test_colsum_blocks_match_whole():
    g = torch.Generator().manual_seed(25)
    X = _bf16(1001, 24, g=g)
    init = torch.randn(24, generator=g)
    s, b = EB.colsum(X, init, 10, block_rows=1 << 20)
    sc, bc = EB.colsum(X, init, 10, block_rows=97)
    _close(sc, s)
    _close(bc, b)
