"""Row kernels (embedding, LayerNorm, column sums, bar-NLL, GP sampler) vs the CPU oracle."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L
from oracle import pfn_oracle as O


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("T,B,F,E,sep", [(10, 4, 1, 128, 4), (7, 3, 5, 96, 0), (9, 2, 18, 512, 9), (5, 5, 3, 40, 2)])
def test_embed_fwd_bwd(cuda_device, dtype, T, B, F, E, sep):
    torch.manual_seed(0)
    dev = cuda_device
    x, y = torch.rand(T, B, F, device=dev), torch.randn(T, B, device=dev)
    Wx, bx = torch.randn(E, F, device=dev), torch.randn(E, device=dev)
    wy, by = torch.randn(E, device=dev), torch.randn(E, device=dev)
    out = torch.empty(T * B, E, device=dev, dtype=dtype)
    L.embed_fwd(x, y, Wx, bx, wy, by, out, T, B, F, E, sep)
    xr = x.cpu().double().requires_grad_(False)
    P = [t.cpu().double().requires_grad_(True) for t in (Wx, bx, wy, by)]
    ref = O.embed_ref(xr, y.cpu().double(), P[0], P[1], P[2].unsqueeze(1), P[3], sep)
    tol = 1e-5 if dtype == torch.float32 else 1e-2
    assert (out.float().cpu().double() - ref).abs().max().item() <= tol * ref.abs().max().item()
    dout = torch.randn(T * B, E, device=dev).to(dtype)
    (ref * dout.float().cpu().double()).sum().backward()
    g = [torch.zeros_like(t) for t in (Wx, bx, wy, by)]
    L.embed_bwd(dout, x, y, g[0], g[1], g[2], g[3], T, B, F, E, sep)
    for got, want in zip(g, P):
        w = want.grad if want.grad is not None else torch.zeros_like(want)
        assert (got.cpu().double() - w).abs().max().item() <= 1e-4 * (w.abs().max().item() + 1)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
# 70 001 rows: every warp of the vector kernels' grids walks more than 32 rows (round its ring and past the backward's
# batch of 32 mean/rstd loads), and the rows end in a ragged tail.
@pytest.mark.parametrize("rows,E", [(37, 128), (1000, 512), (64, 1024), (33, 200), (17, 36), (70001, 512), (70001, 1024)])
def test_layernorm_fwd_bwd(cuda_device, dtype, rows, E):
    torch.manual_seed(1)
    dev = cuda_device
    z = (torch.randn(rows, E, device=dev) * 2 + 0.5).to(dtype)
    gamma, beta = torch.randn(E, device=dev), torch.randn(E, device=dev)
    h = torch.empty_like(z)
    mean, rstd = torch.empty(rows, device=dev), torch.empty(rows, device=dev)
    L.layernorm_fwd(z, gamma, beta, h, mean, rstd)
    # the float64 oracle runs on the GPU: on the CPU the largest shapes take too long
    zr = z.double().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    ref = O.layernorm_ref(zr, gr, br)
    tol = 2e-5 if dtype == torch.float32 else 2e-2
    assert (h.double() - ref).abs().max().item() <= tol * ref.abs().max().item()
    dh = torch.randn(rows, E, device=dev).to(dtype)
    (ref * dh.double()).sum().backward()
    dz = torch.empty_like(z)
    dg, db, cs = (torch.zeros(E, device=dev) for _ in range(3))
    L.layernorm_bwd(dh, z, mean, rstd, gamma, dz, dg, db, cs)
    assert (dz.double() - zr.grad).abs().max().item() <= tol * (zr.grad.abs().max().item() + 1e-3)
    assert (dg.double() - gr.grad).abs().max().item() <= 1e-3 * (gr.grad.abs().max().item() + 1)
    assert (db.double() - br.grad).abs().max().item() <= 1e-3 * (br.grad.abs().max().item() + 1)
    ref_cs = dz.float().sum(0)
    assert (cs - ref_cs).abs().max().item() <= 2e-3 * (ref_cs.abs().max().item() + 1)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_colsum(cuda_device, dtype):
    X = torch.randn(3001, 520, device=cuda_device).to(dtype)[:, :515]
    out = torch.ones(515, device=cuda_device)
    L.colsum(X, out)
    ref = X.float().sum(0) + 1
    assert (out - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()


def _borders(n, dev):
    b = torch.sort(torch.randn(n + 1)).values
    return b.to(dev)


@pytest.mark.parametrize("full_support", [False, True])
@pytest.mark.parametrize("n_bars,dtype", [(100, torch.float32), (100, torch.bfloat16), (1000, torch.float32), (7, torch.float32)])
def test_bar_nll(cuda_device, full_support, n_bars, dtype):
    torch.manual_seed(2)
    dev = cuda_device
    rows = 333
    borders = _borders(n_bars, dev)
    lo, hi = borders[0].item(), borders[-1].item()
    y = torch.rand(rows, device=dev) * (hi - lo) + lo
    y[0], y[1] = borders[0], borders[-1]            # edge fix-ups (bar_distribution.py:21-22)
    y[2], y[3] = borders[3], borders[1]             # exactly on inner borders -> left bucket
    if full_support:
        y[4], y[5] = lo - 1.5, hi + 2.0             # outside the support: clamped + half-normal tails
    ld = (n_bars + 7) // 8 * 8 + 8
    logits = (torch.randn(rows, ld, device=dev) * 3).to(dtype)[:, :n_bars]
    nll = torch.empty(rows, device=dev)
    idx = torch.empty(rows, device=dev, dtype=torch.int64)
    lse = torch.empty(rows, device=dev)
    oob = torch.zeros(1, device=dev, dtype=torch.int32)
    L.bar_nll_fwd(logits, y, borders, n_bars, full_support, nll, idx, lse, oob)
    lr = logits.float().cpu().requires_grad_(True)
    ref = O.bar_nll_ref(lr, y.cpu(), borders.cpu(), full_support)
    ref_idx = O.bucket_idx_ref(y.cpu(), borders.cpu())
    if full_support:
        ref_idx = ref_idx.clamp(0, n_bars - 1)
    assert torch.equal(idx.cpu(), ref_idx), "bucket indices must be bit-exact"
    assert oob.item() == 0
    assert (nll.cpu() - ref).abs().max().item() <= 1e-4 * ref.abs().max().item() + 1e-5
    g = torch.randn(rows, device=dev)
    (ref * g.cpu()).sum().backward()
    dl = torch.full((rows, ld), 9.0, device=dev)
    L.bar_nll_bwd(logits, idx, lse, g, dl, n_bars, n_cols_pad=ld)
    assert (dl[:, :n_bars].cpu() - lr.grad).abs().max().item() <= 1e-4
    assert dl[:, n_bars:].abs().max().item() == 0.0
    # standalone bucket lookup
    idx2 = torch.empty_like(idx)
    L.bar_bucket_idx(y, borders, n_bars, idx2)
    assert torch.equal(idx2.cpu(), O.bucket_idx_ref(y.cpu(), borders.cpu()))


def test_bar_nll_out_of_range_counted(cuda_device):
    dev = cuda_device
    borders = torch.linspace(-1, 1, 11, device=dev)
    y = torch.tensor([0.0, 2.0, -3.0, 0.5], device=dev)
    logits = torch.zeros(4, 10, device=dev)
    nll, lse = torch.empty(4, device=dev), torch.empty(4, device=dev)
    idx = torch.empty(4, device=dev, dtype=torch.int64)
    oob = torch.zeros(1, device=dev, dtype=torch.int32)
    L.bar_nll_fwd(logits, y, borders, 10, False, nll, idx, lse, oob)
    assert oob.item() == 2
    assert idx.tolist()[1] == 10 and idx.tolist()[2] == -1


@pytest.mark.parametrize("kernel,code", [("rbf", L.KERNEL_RBF), ("matern52", L.KERNEL_MATERN52), ("matern32", L.KERNEL_MATERN32), ("matern12", L.KERNEL_MATERN12)])
@pytest.mark.parametrize("Bn,T,F,noise", [(3, 50, 1, 0.1), (2, 130, 5, 0.05), (2, 257, 2, 0.1), (1, 31, 3, 0.2)])
def test_gp_sample_matches_lapack(cuda_device, kernel, code, Bn, T, F, noise):
    torch.manual_seed(3)
    dev = cuda_device
    x = torch.rand(Bn, T, F, device=dev)
    z = torch.randn(Bn, T, device=dev)
    ls = torch.rand(Bn, F, device=dev) * 0.5 + 0.1
    os_ = torch.rand(Bn, device=dev) + 0.5
    nz = torch.full((Bn,), noise, device=dev)
    ldw = (T + 3) // 4 * 4
    y = torch.empty(Bn, T, device=dev)
    work = torch.empty(Bn, T, ldw, device=dev)
    info = torch.full((Bn,), -1, device=dev, dtype=torch.int32)
    L.gp_sample(x, z, ls, os_, nz, 0.0, code, y, work, info)
    yr, Lr = O.gp_sample_ref(x.cpu().double(), z.cpu().double(), ls.cpu().double(), os_.cpu().double(), nz.cpu().double(), kernel)
    assert info.tolist() == [0] * Bn
    Lg = torch.tril(work[:, :, :T].transpose(1, 2).cpu().double())     # the kernel keeps the factor transposed
    K = O.gp_kernel_ref(x.cpu().double(), ls.cpu().double(), os_.cpu().double(), nz.cpu().double(), kernel)
    resid = (Lg @ Lg.transpose(-1, -2) - K).abs().max().item()
    assert resid <= 2e-5 * K.abs().max().item(), f"L L^T residual {resid}"
    assert (y.cpu().double() - yr).abs().max().item() <= 5e-3 * yr.abs().max().item()


def test_gp_sample_flags_non_pd(cuda_device):
    dev = cuda_device
    T = 40
    x = torch.zeros(1, T, 1, device=dev)            # identical inputs, zero noise -> singular K
    z = torch.randn(1, T, device=dev)
    one = torch.ones(1, device=dev)
    y = torch.empty(1, T, device=dev)
    work = torch.empty(1, T, T, device=dev)
    info = torch.zeros(1, device=dev, dtype=torch.int32)
    L.gp_sample(x, z, one.view(1, 1), one, torch.zeros(1, device=dev), 0.0, L.KERNEL_RBF, y, work, info)
    assert info.item() > 0
