"""Row kernels (embedding, LayerNorm, column sums, bar-NLL, GP sampler) vs the CPU oracle.

The embedding, LayerNorm, column-sum and bar-NLL results are held element by element to the fp64 bounds of
oracle/error_budget.py (|got - exact| <= c (u M + E)); the fp64 work runs on the GPU."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L
from transformerscandobayesianinference_b200.engine import LN_EPS
from oracle import error_budget as EB, pfn_oracle as O


def _u(dtype):
    return EB.U32 if dtype == torch.float32 else EB.U


def _aligned(*ts):
    return all(t.data_ptr() % 16 == 0 for t in ts)


def _check_embed(dev, dtype, T, B, F, E, sep, tag):
    x, y = torch.rand(T, B, F, device=dev), torch.randn(T, B, device=dev)
    Wx, bx = torch.randn(E, F, device=dev), torch.randn(E, device=dev)
    wy, by = torch.randn(E, device=dev), torch.randn(E, device=dev)
    out = torch.empty(T * B, E, device=dev, dtype=dtype)
    L.embed_fwd(x, y, Wx, bx, wy, by, out, T, B, F, E, sep)
    rows = T * B
    exact, bound = EB.embed_fwd(x.reshape(rows, F), y.reshape(rows), Wx, bx, wy, by, sep * B, _u(dtype))
    EB.check(f"embed_fwd{tag}", out, exact, bound, EB.C_EMBED)
    dout = torch.randn(T * B, E, device=dev).to(dtype)
    g = [torch.zeros_like(t) for t in (Wx, bx, wy, by)]
    L.embed_bwd(dout, x, y, g[0], g[1], g[2], g[3], T, B, F, E, sep)
    ref = EB.embed_bwd(dout, x.reshape(rows, F), y.reshape(rows), sep * B, EB.embed_bwd_depth(rows))
    for got, name in zip(g, ("dWx", "dbx", "dwy", "dby")):
        EB.check(f"embed_bwd {name}{tag}", got, ref[name][0].reshape(got.shape), ref[name][1].reshape(got.shape), EB.C_ROWSUM)


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
    # the exact value is also the reference's (autograd of the oracle); the bounds come from oracle/error_budget.py
    xr = x.cpu().double()
    P = [t.cpu().double().requires_grad_(True) for t in (Wx, bx, wy, by)]
    ref = O.embed_ref(xr, y.cpu().double(), P[0], P[1], P[2].unsqueeze(1), P[3], sep)
    rows = T * B
    exact, bound = EB.embed_fwd(x.reshape(rows, F), y.reshape(rows), Wx, bx, wy, by, sep * B, _u(dtype))
    assert torch.allclose(exact.cpu(), ref.detach(), rtol=0, atol=1e-12)
    EB.check("embed_fwd", out, exact, bound, EB.C_EMBED)
    dout = torch.randn(T * B, E, device=dev).to(dtype)
    (ref * dout.float().cpu().double()).sum().backward()
    g = [torch.zeros_like(t) for t in (Wx, bx, wy, by)]
    L.embed_bwd(dout, x, y, g[0], g[1], g[2], g[3], T, B, F, E, sep)
    eb = EB.embed_bwd(dout, x.reshape(rows, F), y.reshape(rows), sep * B, EB.embed_bwd_depth(rows))
    for got, want, name in zip(g, P, ("dWx", "dbx", "dwy", "dby")):
        w = want.grad if want.grad is not None else torch.zeros_like(want)
        assert torch.allclose(eb[name][0].reshape(got.shape).cpu(), w, rtol=0, atol=1e-9)
        EB.check(f"embed_bwd {name}", got, eb[name][0].reshape(got.shape), eb[name][1].reshape(got.shape), EB.C_ROWSUM)


# more than 512 rows, so that embed_bwd reduces across CTAs (ragged last CTA); F covers one and several f0 launches with
# ragged last groups; sep = 0 (no train rows) and sep = T (all train rows)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("F", [1, 8, 9, 64, 100])
@pytest.mark.parametrize("sep", [0, 150, 300])
def test_embed_across_ctas(cuda_device, dtype, F, sep):
    torch.manual_seed(F + sep)
    _check_embed(cuda_device, dtype, 300, 4, F, 256, sep, f" T=300 B=4 F={F} sep={sep}")


def _ln_check(dev, z, h, dh, dz, tag, init=None):
    """LayerNorm forward and backward of z (already laid out: views, strides) against the fp64 bounds."""
    rows, E = z.shape
    dtype = z.dtype
    u = _u(dtype)
    gamma, beta = torch.randn(E, device=dev), torch.randn(E, device=dev)
    mean, rstd = torch.empty(rows, device=dev), torch.empty(rows, device=dev)
    L.layernorm_fwd(z, gamma, beta, h, mean, rstd, eps=LN_EPS)
    f = EB.layernorm_fwd(z, gamma, beta, u, eps=LN_EPS)
    EB.check(f"layernorm h{tag}", h, f["h"], f["h_bound"], EB.C_LN)
    EB.check(f"layernorm mean{tag}", mean, f["mean"], f["mean_bound"], EB.C_LN)
    EB.check(f"layernorm rstd{tag}", rstd, f["rstd"], f["rstd_bound"], EB.C_LN)
    cols = [torch.zeros(E, device=dev) if init is None else init[i].clone() for i in range(3)]
    L.layernorm_bwd(dh, z, mean, rstd, gamma, dz, cols[0], cols[1], cols[2])
    vec = EB.ln_vec(E, [z.stride(0), dh.stride(0), dz.stride(0)], _aligned(z, dh, dz, gamma))
    depth = EB.ln_bwd_colsum_depth(rows, E, z.element_size(), vec, L.num_sms())
    b = EB.layernorm_bwd(dh, z, gamma, mean, rstd, u, depth, init, eps=LN_EPS)
    EB.check(f"layernorm dz{tag}", dz, b["dz"], b["dz_bound"], EB.C_LN_GRAD)
    for got, name in zip(cols, ("dgamma", "dbeta", "colsum")):
        EB.check(f"layernorm {name}{tag}", got, b[name], b[name + "_bound"], EB.C_LN_GRAD)
    return f, b


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
# 70 001 rows: every warp of the vector kernels' grids walks more than 32 rows (round its ring and past the backward's
# batch of 32 mean/rstd loads), and the rows end in a ragged tail.
@pytest.mark.parametrize("rows,E", [(37, 128), (1000, 512), (64, 1024), (33, 200), (17, 36), (70001, 512), (70001, 1024)])
def test_layernorm_fwd_bwd(cuda_device, dtype, rows, E):
    torch.manual_seed(1)
    dev = cuda_device
    z = (torch.randn(rows, E, device=dev) * 2 + 0.5).to(dtype)
    h, dz = torch.empty_like(z), torch.empty_like(z)
    dh = torch.randn(rows, E, device=dev).to(dtype)
    # the float64 oracle runs on the GPU: on the CPU the largest shapes take too long
    f, b = _ln_check(dev, z, h, dh, dz, f" rows={rows} E={E}")
    if rows <= 1000:                    # the helpers' exact values are the reference LayerNorm and its autograd
        zr = z.double().requires_grad_(True)
        ref = O.layernorm_ref(zr, torch.ones(E, device=dev, dtype=torch.float64), torch.zeros(E, device=dev, dtype=torch.float64))
        g1 = EB.layernorm_fwd(z, torch.ones(E, device=dev), torch.zeros(E, device=dev), _u(dtype))
        assert torch.allclose(g1["h"], ref.detach(), rtol=0, atol=1e-10)
        (ref * dh.double()).sum().backward()
        b1 = EB.layernorm_bwd(dh, z, torch.ones(E, device=dev), g1["mean"].float(), g1["rstd"].float(), _u(dtype), 1)
        assert torch.allclose(b1["dz"], zr.grad, rtol=0, atol=1e-8)


def _ln_layout(dev, dtype, rows, E, ld, offset):
    """Three [rows, E] tensors with row stride ld whose data start `offset` elements into their buffers."""
    def one():
        buf = torch.empty(rows * ld + offset + 8, device=dev, dtype=dtype)
        return buf[offset:offset + rows * ld].view(rows, ld)[:, :E]
    return one(), one(), one()


# name, rows, E, dtype, data mean, data std, row stride pad, element offset, non-zero initial column sums
LN_CASES = [
    ("vec1", 300, 256, torch.bfloat16, 0.5, 2.0, 0, 0, True),
    ("vec2_ragged", 300, 264, torch.float32, 0.5, 2.0, 0, 0, True),
    ("vec4_ragged", 300, 776, torch.bfloat16, 0.5, 2.0, 0, 0, False),
    ("generic_E36", 500, 36, torch.bfloat16, 0.5, 2.0, 0, 0, True),
    ("generic_E100", 500, 100, torch.float32, 0.5, 2.0, 0, 0, False),
    ("generic_E1536", 700, 1536, torch.bfloat16, 0.5, 2.0, 0, 0, True),
    ("generic_E2048", 700, 2048, torch.float32, 0.5, 2.0, 0, 0, False),
    ("generic_unaligned", 333, 512, torch.float32, 0.5, 2.0, 0, 1, True),
    ("generic_unaligned_bf16", 333, 512, torch.bfloat16, 0.5, 2.0, 0, 1, False),
    ("vec_strided", 1000, 512, torch.bfloat16, 0.5, 2.0, 24, 0, True),
    ("vec_strided_fp32", 1000, 256, torch.float32, 0.5, 2.0, 8, 0, False),
    ("one_row_E8", 1, 8, torch.float32, 0.5, 2.0, 0, 0, True),
    ("one_row_E8_bf16", 1, 8, torch.bfloat16, 0.5, 2.0, 0, 0, False),
    ("mean1e3_std1", 2000, 512, torch.float32, 1e3, 1.0, 0, 0, True),
    ("mean1e3_std1_generic", 500, 100, torch.float32, 1e3, 1.0, 0, 0, False),
    ("mean64_bf16", 2000, 512, torch.bfloat16, 64.0, 1.0, 0, 0, True),
    ("std3e-3_eps", 2000, 512, torch.float32, 0.2, 3e-3, 0, 0, False),
    ("std3e-3_eps_bf16", 2000, 128, torch.bfloat16, 0.0, 3e-3, 0, 0, True),
    ("constant_rows", 300, 512, torch.float32, 0.1, 0.0, 0, 0, True),
    ("constant_rows_bf16", 300, 1024, torch.bfloat16, -3.0, 0.0, 0, 0, False),
]


@pytest.mark.parametrize("name,rows,E,dtype,mu,sd,pad,offset,init", LN_CASES, ids=[c[0] for c in LN_CASES])
def test_layernorm_paths_and_edges(cuda_device, name, rows, E, dtype, mu, sd, pad, offset, init):
    """Every dispatch path (vector kernels with one, two and four 256-column chunks per lane; the generic kernel for
    E % 8 != 0, E > 1024 and pointers that are not 16-byte aligned), strided views, one-row problems, and rows whose
    mean dwarfs their spread, whose variance is near eps or is zero; the column sums accumulate into non-zero values."""
    torch.manual_seed(len(name) + rows)
    dev = cuda_device
    z, h, dz = _ln_layout(dev, dtype, rows, E, E + pad, offset)
    z.copy_((torch.randn(rows, E, device=dev) * sd + mu).to(dtype))
    dh = _ln_layout(dev, dtype, rows, E, E + pad, offset)[0]
    dh.copy_(torch.randn(rows, E, device=dev).to(dtype))
    init_cols = [torch.randn(E, device=dev) * 10 for _ in range(3)] if init else None
    _ln_check(dev, z, h, dh, dz, f" {name}", init_cols)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_colsum(cuda_device, dtype):
    X = torch.randn(3001, 520, device=cuda_device).to(dtype)[:, :515]
    out = torch.ones(515, device=cuda_device)
    init = out.clone()
    L.colsum(X, out)
    exact, bound = EB.colsum(X, init, EB.colsum_depth(3001, 515, 520, X.element_size(), L.num_sms()))
    EB.check("colsum 3001x515", out, exact, bound, EB.C_ROWSUM)


# N covers colsum_vec_kernel with NV = 1 (8, 256), NV = 2 (264, 512), NV = 4 in one group (1000) and in several groups
# with a ragged last one (1536, 2056), and the generic kernel (515, ld not a multiple of 8); rows from 1 to the engine's
# T * B = 512 000 at cfg 2 (bias gradients of the 512-, 1024- and 1536-wide layers)
COLSUM_CASES = [(1, 8, 0), (7, 256, 8), (3001, 264, 8), (1000, 512, 0), (4099, 1000, 24), (20000, 1536, 0),
                (777, 2056, 8), (2, 515, 5), (70001, 515, 1), (512000, 512, 0), (512000, 1024, 0), (512000, 1536, 0)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("rows,N,pad", COLSUM_CASES)
def test_colsum_paths(cuda_device, dtype, rows, N, pad):
    torch.manual_seed(rows + N)
    dev = cuda_device
    # a positive mean keeps the column sums from cancelling, so a rounding slip in the running sums shows
    X = (torch.rand(rows, N + pad, device=dev) + 0.25 * torch.randn(rows, N + pad, device=dev)).to(dtype)[:, :N]
    out = torch.randn(N, device=dev) * 100
    init = out.clone()
    L.colsum(X, out)
    exact, bound = EB.colsum(X, init, EB.colsum_depth(rows, N, N + pad, X.element_size(), L.num_sms(), _aligned(X)))
    EB.check(f"colsum {rows}x{N} ld={N + pad}", out, exact, bound, EB.C_ROWSUM)


def _borders(n, dev):
    b = torch.sort(torch.randn(n + 1)).values
    return b.to(dev)


def _bar_check(logits, y, borders, n_bars, full_support, tag, d_dtype=torch.float32, pad=None, ld_d=None, rows_nan=()):
    """pfn_bar_nll_fwd / bwd on `logits` against the fp64 bounds; rows_nan: rows whose nll must be NaN (all -inf)."""
    dev = logits.device
    rows = logits.shape[0]
    nll = torch.empty(rows, device=dev)
    idx = torch.empty(rows, device=dev, dtype=torch.int64)
    lse = torch.empty(rows, device=dev)
    oob = torch.zeros(1, device=dev, dtype=torch.int32)
    L.bar_nll_fwd(logits, y, borders, n_bars, full_support, nll, idx, lse, oob)
    f = EB.bar_nll_fwd(logits, y, borders, full_support)
    assert torch.equal(idx, f["idx"]), "bucket indices must be bit-exact"
    assert oob.item() == 0
    ok = torch.ones(rows, dtype=torch.bool, device=dev)
    for r in rows_nan:
        assert math.isnan(nll[r].item()) and lse[r].item() == float("-inf")
        ok[r] = False
    EB.check(f"bar_nll lse{tag}", lse[ok], f["lse"][ok], f["lse_bound"][ok], EB.C_BAR)
    EB.check(f"bar_nll nll{tag}", nll[ok], f["nll"][ok], f["nll_bound"][ok], EB.C_BAR)
    g = torch.randn(rows, device=dev)
    pad = (n_bars + 7) // 8 * 8 if pad is None else pad
    ld_d = pad if ld_d is None else ld_d
    dl = torch.full((rows, ld_d), 9.0, device=dev).to(d_dtype)
    L.bar_nll_bwd(logits, idx, lse, g, dl, n_bars, n_cols_pad=pad)
    exact, bound = EB.bar_nll_bwd(logits[ok], idx[ok], lse[ok], g[ok], _u(d_dtype))
    EB.check(f"bar_nll dlogits{tag}", dl[ok, :n_bars], exact, bound, EB.C_BAR_GRAD)
    assert (dl[:, n_bars:pad] == 0).all(), "padding columns must be zero"
    if ld_d > pad:
        assert (dl[:, pad:].float() == 9.0).all(), "columns beyond n_cols_pad must not be written"
    return idx


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
    idx = _bar_check(logits, y, borders, n_bars, full_support, f" n={n_bars}", pad=ld)
    ref_idx = O.bucket_idx_ref(y.cpu(), borders.cpu())
    if full_support:
        ref_idx = ref_idx.clamp(0, n_bars - 1)
    assert torch.equal(idx.cpu(), ref_idx), "bucket indices must be bit-exact"
    # the helper's exact nll is the reference's
    ref = O.bar_nll_ref(logits.double().cpu(), y.cpu().double(), borders.cpu().double(), full_support)
    assert torch.allclose(EB.bar_nll_fwd(logits, y, borders, full_support)["nll"].cpu(), ref, rtol=1e-12, atol=1e-12)
    # standalone bucket lookup
    idx2 = torch.empty_like(idx)
    L.bar_bucket_idx(y, borders, n_bars, idx2)
    assert torch.equal(idx2.cpu(), O.bucket_idx_ref(y.cpu(), borders.cpu()))


PAIRS = [(torch.float32, torch.float32), (torch.float32, torch.bfloat16), (torch.bfloat16, torch.float32),
         (torch.bfloat16, torch.bfloat16)]


def _bar_targets(rows, borders, full_support, g):
    """Targets spread over the support, on borders, and (full support) deep in both half-normal tails."""
    n = borders.numel() - 1
    lo, hi = borders[0].item(), borders[-1].item()
    y = (torch.rand(rows, generator=g) * (hi - lo) + lo).clamp(lo, hi)
    y[:8] = borders[torch.randint(0, n + 1, (8,), generator=g)].cpu()
    if full_support:
        w0, w1 = (borders[1] - borders[0]).item(), (borders[-1] - borders[-2]).item()
        y[8:40] = lo - w0 * torch.rand(32, generator=g) * 40
        y[40:72] = hi + w1 * torch.rand(32, generator=g) * 40
    return y


# rows beyond num_sms * 64, so that every warp of the grid loops; the dtype pair (logits, dlogits) cycles over the four
# the ABI exports
@pytest.mark.parametrize("full_support", [False, True])
@pytest.mark.parametrize("n_bars", [2, 7, 31, 32, 33, 100, 1000])
def test_bar_nll_shapes(cuda_device, n_bars, full_support):
    dev = cuda_device
    g = torch.Generator().manual_seed(n_bars + 7 * full_support)
    rows = 20011 if n_bars < 1000 else 9001
    dtype, d_dtype = PAIRS[(n_bars + full_support) % 4]
    borders = torch.sort(torch.randn(n_bars + 1, generator=g)).values.to(dev)
    y = _bar_targets(rows, borders, full_support, g).to(dev)
    logits = (torch.randn(rows, n_bars, generator=g) * 3).to(dev).to(dtype)
    _bar_check(logits, y, borders, n_bars, full_support, f" n={n_bars} fs={int(full_support)} {dtype}->{d_dtype}", d_dtype)


@pytest.mark.parametrize("dtype,d_dtype", PAIRS)
def test_bar_nll_dtype_pairs_and_wide_dlogits(cuda_device, dtype, d_dtype):
    """All four (logits, dlogits) pairs, logits with a row stride, dlogits rows wider than n_cols_pad; n_bars = 2 with
    full support (both buckets are tails)."""
    dev = cuda_device
    g = torch.Generator().manual_seed(31)
    for n_bars, full_support in [(100, True), (2, True)]:
        rows = 10007
        borders = torch.sort(torch.randn(n_bars + 1, generator=g)).values.to(dev)
        y = _bar_targets(rows, borders, full_support, g).to(dev)
        logits = (torch.randn(rows, n_bars + 13, generator=g) * 3).to(dev).to(dtype)[:, :n_bars]
        pad = (n_bars + 7) // 8 * 8
        _bar_check(logits, y, borders, n_bars, full_support, f" n={n_bars} {dtype}->{d_dtype} ld_d>pad", d_dtype,
                   pad=pad, ld_d=pad + 24)


@pytest.mark.parametrize("full_support", [False, True])
def test_bar_nll_narrow_buckets_far_out(cuda_device, full_support):
    """Buckets of width ~1e-3 around 1000 (widths of 16 fp32 ulps) and around -3000."""
    dev = cuda_device
    g = torch.Generator().manual_seed(41)
    for base in (1000.0, -3000.0):
        widths = (torch.rand(100, generator=g) + 0.1) * 1e-3
        borders = (base + torch.cat([torch.zeros(1, dtype=torch.float64), torch.cumsum(widths.double(), 0)])).float()
        borders = torch.unique(borders).to(dev)          # sorted, distinct after the fp32 rounding
        n_bars = borders.numel() - 1
        y = _bar_targets(20011, borders, full_support, g).to(dev)
        logits = (torch.randn(20011, n_bars, generator=g) * 3).to(dev)
        _bar_check(logits, y, borders, n_bars, full_support, f" narrow@{base:g} fs={int(full_support)}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_bar_nll_neg_inf_logits(cuda_device, dtype):
    """-inf logits (a bar the model rules out) add nothing to the log-sum-exp, as in log_softmax: in a lane's first bar
    (bars 0 and 5, the first of lanes 0 and 5), in later bars, in every bar of a lane, and in a whole row (nll NaN, lse
    -inf, as torch gives)."""
    dev = cuda_device
    g = torch.Generator().manual_seed(51)
    n_bars, rows = 100, 4099
    borders = torch.sort(torch.randn(n_bars + 1, generator=g)).values.to(dev)
    y = _bar_targets(rows, borders, True, g).to(dev)
    idx = EB.bucket_index(y, borders).clamp(0, n_bars - 1)
    logits = (torch.randn(rows, n_bars, generator=g) * 3).to(dev)
    ninf = torch.zeros(rows, n_bars, dtype=torch.bool, device=dev)
    ninf[:, 5] = True
    ninf[::2, 0] = True
    ninf[::3, 40] = True
    ninf[1::7, 7::32] = True                              # every bar of lane 7
    ninf[::5, 60:] = True
    ninf[torch.arange(rows, device=dev), idx] = False     # the target's bar stays finite ...
    ninf[17] = True                                       # ... except in one row that is -inf throughout
    logits = logits.masked_fill(ninf, float("-inf")).to(dtype)
    ref = torch.log_softmax(logits.double(), -1)
    assert torch.isfinite(ref[:17].gather(1, idx[:17].unsqueeze(1))).all()
    _bar_check(logits, y, borders, n_bars, True, f" -inf {dtype}", rows_nan=(17,))


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
    assert info.tolist() == [0] * Bn
    Lg = EB.gp_factor(work, T)                  # the kernel keeps the factor transposed
    assert (torch.diagonal(Lg, dim1=1, dim2=2) > 0).all()
    K, E_K = EB.gp_kernel(x, ls, os_, nz, 0.0, code)
    LLt, bound = EB.gp_factor_residual(Lg, E_K)
    EB.check(f"gp factor {kernel} T={T}", LLt, K, bound, EB.C_GP_FACTOR)
    ye, yb = EB.gp_draw(Lg, z)
    EB.check(f"gp y {kernel} T={T}", y, ye, yb, EB.C_GP_Y)
    # the oracle's kernel matrix and LAPACK's draw (well conditioned here: noise >= 0.05)
    Kr = O.gp_kernel_ref(x.cpu().double(), ls.cpu().double(), os_.cpu().double(), nz.cpu().double(), kernel)
    assert torch.allclose(K.cpu(), Kr, rtol=1e-12, atol=1e-15)
    yr, Lr = O.gp_sample_ref(x.cpu().double(), z.cpu().double(), ls.cpu().double(), os_.cpu().double(), nz.cpu().double(), kernel)
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
