"""The row-kernel bounds of oracle/error_budget.py (LayerNorm, column sums, embedding, bar NLL, Adam) on float32 CPU
restatements of the kernels that round where the kernels round: a correct restatement lies inside them at c = 1, and
each numerical slip a kernel could make falls outside them at the constant the GPU tests use.  Each slip also reports
whether the max-scaled tolerances the GPU tests used before pass it."""
import math

import pytest
import torch

from oracle import error_budget as EB

F32 = torch.float32
NUM_SMS = 132                      # H100 SXM


def _fma(a, b, c):
    """fp32 fma: the product of two fp32 values is exact in fp64, so one rounding of the fp64 sum."""
    return (a.double() * b.double() + c.double()).float()


def _warp_sum(x):
    """The 5-level xor butterfly over the last dim (32 lanes), in fp32."""
    for o in (16, 8, 4, 2, 1):
        x = x + x[..., torch.arange(32) ^ o]
    return x[..., 0]


def _ratio(got, exact, bound):
    err = (got.double() - exact.double()).abs()
    return (err / bound.double().clamp_min(1e-300)).masked_fill(bound == 0, 0.0).max().item()


def _report(name, ratio, c, old):
    print(f"[perturbation] {name}: err/bound {ratio:.3g} (c {c}); old max-scaled tolerance {'PASSES' if old else 'fails'}")


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm (the generic kernel's order: lane i sums columns i, i + 32, ...; then the butterfly)
# ------------------------------------------------------------------------------------------------------------------
def ln_fwd(z, gamma, beta, out_dtype, eps=1e-5, one_pass=False, eps_after=False, unbiased=False):
    rows, E = z.shape
    zp = torch.cat([z.float(), torch.zeros(rows, (-E) % 32)], 1).view(rows, -1, 32)
    valid = (torch.arange(zp.shape[1] * 32) < E).view(-1, 32)
    s = torch.zeros(rows, 32)
    for j in range(zp.shape[1]):
        s = torch.where(valid[j], s + zp[:, j], s)
    mean = _warp_sum(s) / E
    ss = torch.zeros(rows, 32)
    for j in range(zp.shape[1]):
        d = zp[:, j] if one_pass else zp[:, j] - mean.unsqueeze(1)
        ss = torch.where(valid[j], _fma(d, d, ss), ss)
    var = _warp_sum(ss) / E
    if one_pass:
        var = var - mean * mean
    if unbiased:
        var = var * E / (E - 1)
    rstd = 1.0 / (torch.sqrt(var) + eps) if eps_after else torch.rsqrt(var + eps)
    h = _fma((z.float() - mean.unsqueeze(1)) * rstd.unsqueeze(1), gamma.float(), beta.float()).to(out_dtype)
    return h, mean, rstd


def ln_bwd(dh, z, mean, rstd, gamma):
    E = z.shape[1]
    xh = (z.float() - mean.unsqueeze(1)) * rstd.unsqueeze(1)
    g = dh.float() * gamma.float()
    s1, s2 = g.sum(1, keepdim=True) / E, (g * xh).sum(1, keepdim=True) / E
    o = rstd.unsqueeze(1) * (g - s1 - xh * s2)
    cols = []
    for t in (dh.float() * xh, dh.float(), o):      # one atomic per row in row order (the generic kernel)
        acc = torch.zeros(E)
        for r in range(t.shape[0]):
            acc = acc + t[r]
        cols.append(acc)
    return o.to(z.dtype), cols


def _ln_data(rows, E, mu, sd, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    z = (torch.randn(rows, E, generator=g, dtype=torch.float64) * sd + mu).to(dtype)
    return z, torch.randn(E, generator=g), torch.randn(E, generator=g)


@pytest.mark.parametrize("rows,E,mu,sd,dtype", [(64, 512, 0.5, 2.0, F32), (64, 100, 1e3, 1.0, F32), (64, 36, 0.5, 2.0, torch.bfloat16),
                                               (64, 512, 64.0, 1.0, torch.bfloat16), (64, 512, 0.2, 3e-3, F32), (8, 512, 0.1, 0.0, F32)])
def test_layernorm_restatement_inside_bound_at_c1(rows, E, mu, sd, dtype):
    z, gamma, beta = _ln_data(rows, E, mu, sd, dtype, E + rows)
    u = EB.U32 if dtype == F32 else EB.U
    h, mean, rstd = ln_fwd(z, gamma, beta, dtype)
    f = EB.layernorm_fwd(z, gamma, beta, u)
    EB.check("host layernorm h", h, f["h"], f["h_bound"], 1.0)
    EB.check("host layernorm mean", mean, f["mean"], f["mean_bound"], 1.0)
    EB.check("host layernorm rstd", rstd, f["rstd"], f["rstd_bound"], 1.0)
    dh = torch.randn(rows, E, generator=torch.Generator().manual_seed(1)).to(dtype)
    dz, cols = ln_bwd(dh, z, mean, rstd, gamma)
    b = EB.layernorm_bwd(dh, z, gamma, mean, rstd, u, EB.ln_bwd_colsum_depth(rows, E, z.element_size(), False, NUM_SMS))
    EB.check("host layernorm dz", dz, b["dz"], b["dz_bound"], 1.0)
    for got, name in zip(cols, ("dgamma", "dbeta", "colsum")):
        EB.check(f"host layernorm {name}", got, b[name], b[name + "_bound"], 1.0)


# name, data (rows, E, mean, std, dtype), slip, whether the old tolerance (2e-5 max|h| fp32, 2e-2 max|h| bf16) passes it
LN_SLIPS = [
    ("one_pass_variance", (64, 512, 1e3, 1.0, F32), dict(one_pass=True), False),
    ("eps_after_rsqrt", (64, 512, 0.2, 3e-3, F32), dict(eps_after=True), False),
    ("unbiased_variance_bf16", (64, 36, 0.5, 2.0, torch.bfloat16), dict(unbiased=True), True),
]


@pytest.mark.parametrize("name,data,kw,old_passes", LN_SLIPS, ids=[s[0] for s in LN_SLIPS])
def test_layernorm_slip_outside_bound(name, data, kw, old_passes):
    rows, E, mu, sd, dtype = data
    z, gamma, beta = _ln_data(rows, E, mu, sd, dtype, 3)
    u = EB.U32 if dtype == F32 else EB.U
    f = EB.layernorm_fwd(z, gamma, beta, u)
    h, _, _ = ln_fwd(z, gamma, beta, dtype, **kw)
    r = _ratio(h, f["h"], f["h_bound"])
    tol = 2e-5 if dtype == F32 else 2e-2
    old = (h.double() - f["h"]).abs().max().item() <= tol * f["h"].abs().max().item()
    _report(f"layernorm {name}", r, EB.C_LN, old)
    assert r > EB.C_LN
    assert old == old_passes


# ------------------------------------------------------------------------------------------------------------------
# column sums: colsum_vec_kernel's order (warp w owns rows w, w + nwarps, ...; 8 warps per CTA; one atomic per CTA)
# ------------------------------------------------------------------------------------------------------------------
def colsum_vec(X, init, num_sms, bf16_acc=False, drop_last=False):
    rows, N = X.shape
    grid = min(num_sms * 4, -(-rows // 8))
    nwarps = grid * 8
    Xf = X.float()
    if drop_last:
        Xf = Xf[:-1]
    pad = (-Xf.shape[0]) % nwarps
    Xw = torch.cat([Xf, torch.zeros(pad, N)]).view(-1, nwarps, N)        # [steps, warp, N]
    acc = torch.zeros(nwarps, N)
    for j in range(Xw.shape[0]):
        acc = acc + Xw[j]
        if bf16_acc:
            acc = acc.to(torch.bfloat16).float()
    out = init.float().clone()
    for cta in acc.view(grid, 8, N):
        s = torch.zeros(N)
        for w in range(8):
            s = s + cta[w]
        out = out + s
    return out


def test_colsum_restatement_inside_bound_at_c1():
    g = torch.Generator().manual_seed(5)
    for rows, N in [(1, 8), (3001, 264), (60000, 256)]:
        X = (torch.rand(rows, N, generator=g) + 0.25 * torch.randn(rows, N, generator=g))
        init = torch.randn(N, generator=g) * 100
        exact, bound = EB.colsum(X, init, EB.colsum_depth(rows, N, N, 4, NUM_SMS))
        EB.check(f"host colsum {rows}x{N}", colsum_vec(X, init, NUM_SMS), exact, bound, 1.0)


# old: 1e-3 max|ref|
@pytest.mark.parametrize("name,kw,old_passes", [("bf16_partials", dict(bf16_acc=True), True),
                                                ("dropped_last_row", dict(drop_last=True), True)])
def test_colsum_slip_outside_bound(name, kw, old_passes):
    g = torch.Generator().manual_seed(6)
    rows, N = 60001, 256
    X = torch.rand(rows, N, generator=g) + 0.25 * torch.randn(rows, N, generator=g)
    init = torch.zeros(N)
    exact, bound = EB.colsum(X, init, EB.colsum_depth(rows, N, N, 4, NUM_SMS))
    got = colsum_vec(X, init, NUM_SMS, **kw)
    r = _ratio(got, exact, bound)
    old = (got.double() - exact).abs().max().item() <= 1e-3 * exact.abs().max().item()
    _report(f"colsum {name}", r, EB.C_ROWSUM, old)
    assert r > EB.C_ROWSUM
    assert old == old_passes


# ------------------------------------------------------------------------------------------------------------------
# embedding
# ------------------------------------------------------------------------------------------------------------------
def embed_fwd(x, y, Wx, bx, wy, by, train_rows):
    acc = bx.expand(x.shape[0], -1).clone()
    for f in range(x.shape[1]):
        acc = _fma(x[:, f:f + 1], Wx[:, f].unsqueeze(0), acc)
    t = (torch.arange(x.shape[0]) < train_rows).unsqueeze(1)
    return torch.where(t, acc + _fma(y.unsqueeze(1), wy.unsqueeze(0), by.unsqueeze(0)), acc)


def embed_bwd(dout, x, y, train_rows, drop_last=False):
    rows, E = dout.shape
    d = dout.float()
    out = {k: 0 for k in ("dWx", "dbx", "dwy", "dby")}
    last = rows - 1 if drop_last else rows
    for r0 in range(0, rows, 512):                       # one CTA per 512 rows, serial inside, atomics across
        sWx, sd, sdt, sdy = torch.zeros(E, x.shape[1]), torch.zeros(E), torch.zeros(E), torch.zeros(E)
        for r in range(r0, min(r0 + 512, last)):
            sd = sd + d[r]
            if r < train_rows:
                sdt = sdt + d[r]
                sdy = _fma(d[r], y[r].expand(E), sdy)
            sWx = _fma(d[r].unsqueeze(1), x[r].unsqueeze(0), sWx)
        for k, v in (("dWx", sWx), ("dbx", sd), ("dwy", sdy), ("dby", sdt)):
            out[k] = out[k] + v
    return out


def _embed_data(rows, F, E, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(rows, F, generator=g), torch.randn(rows, generator=g), torch.randn(E, F, generator=g),
            torch.randn(E, generator=g), torch.randn(E, generator=g), torch.randn(E, generator=g),
            torch.randn(rows, E, generator=g).to(torch.bfloat16))


def test_embed_restatement_inside_bound_at_c1():
    rows, F, E, train = 1201, 9, 64, 600
    x, y, Wx, bx, wy, by, dout = _embed_data(rows, F, E, 7)
    exact, bound = EB.embed_fwd(x, y, Wx, bx, wy, by, train, EB.U32)
    EB.check("host embed_fwd", embed_fwd(x, y, Wx, bx, wy, by, train), exact, bound, 1.0)
    got = embed_bwd(dout, x, y, train)
    ref = EB.embed_bwd(dout, x, y, train, EB.embed_bwd_depth(rows))
    for k in got:
        EB.check(f"host embed_bwd {k}", got[k], ref[k][0], ref[k][1], 1.0)


def test_embed_bwd_dropped_last_row_outside_bound():
    rows, F, E, train = 1201, 9, 64, 1201
    x, y, Wx, bx, wy, by, dout = _embed_data(rows, F, E, 8)
    got = embed_bwd(dout, x, y, train, drop_last=True)
    ref = EB.embed_bwd(dout, x, y, train, EB.embed_bwd_depth(rows))
    r = max(_ratio(got[k], ref[k][0], ref[k][1]) for k in got)
    old = all((got[k].double() - ref[k][0]).abs().max().item() <= 1e-4 * (ref[k][0].abs().max().item() + 1) for k in got)
    _report("embed_bwd dropped_last_row", r, EB.C_ROWSUM, old)
    assert r > EB.C_ROWSUM
    assert not old


# ------------------------------------------------------------------------------------------------------------------
# bar NLL: the forward's lane loop (lane l takes bars l, l + 32, ...) and the backward
# ------------------------------------------------------------------------------------------------------------------
HALF_LOG_2PI_F32 = 0.9189385332046727


def bar_lse(z, lazy=False, skip_neg_inf=True):
    rows, n = z.shape
    steps = -(-n // 32)
    zp = torch.cat([z.float(), torch.zeros(rows, steps * 32 - n)], 1).view(rows, steps, 32)
    m, s = torch.full((rows, 32), float("-inf")), torch.zeros(rows, 32)
    for j in range(steps):
        v = zp[:, j]
        valid = (j * 32 + torch.arange(32)) < n
        up = (v > m) & valid
        corr = torch.exp(m - v)
        if lazy:
            corr = torch.where(corr > 0.98, torch.ones_like(corr), corr)
        s_up = s * corr + 1.0
        add = valid & ~up & ((v != float("-inf")) if skip_neg_inf else torch.ones_like(up))
        s_add = s + torch.exp(v - m)
        s = torch.where(up, s_up, torch.where(add, s_add, s))
        m = torch.where(up, v, m)
    mall = m.amax(1, keepdim=True)
    s = torch.where(m == float("-inf"), torch.zeros_like(s), s * torch.exp(m - mall))
    return mall.squeeze(1) + torch.log(_warp_sum(s))


def bar_nll(z, y, borders, full_support, lse, half_log_2pi=HALF_LOG_2PI_F32):
    n = z.shape[1]
    b = borders.float()
    k = EB.bucket_index(y, borders).clamp(0, n - 1)
    w = b[k + 1] - b[k]
    zk = z.float().gather(1, k.unsqueeze(1)).squeeze(1)
    lp = (zk - lse) - torch.log(w)
    if full_support:
        kI, kL, kH = torch.tensor(EB.ICDF_HALF, dtype=F32), torch.tensor(math.log(2.0), dtype=F32), torch.tensor(half_log_2pi, dtype=F32)
        sc = w / kI
        v0 = torch.clamp(b[1] - y, min=1e-8)
        t0 = (kL - torch.log(sc) - kH - (v0 * v0) / (2.0 * sc * sc)) + torch.log(w)
        v1 = y - b[n - 1]
        t1 = (kL - torch.log(sc) - kH - (v1 * v1) / (2.0 * sc * sc)) + torch.log(w)
        lp = torch.where(k == 0, lp + t0, lp)
        lp = torch.where(k == n - 1, lp + t1, lp)
    return -lp


def _bar_data(rows, n, seed, rising=False):
    g = torch.Generator().manual_seed(seed)
    borders = torch.sort(torch.randn(n + 1, generator=g)).values
    lo, hi = borders[0].item(), borders[-1].item()
    y = (torch.rand(rows, generator=g) * (hi - lo) + lo).clamp(lo, hi)
    w0, w1 = (borders[1] - borders[0]).item(), (borders[-1] - borders[-2]).item()
    y[:32] = lo - w0 * torch.rand(32, generator=g) * 40
    y[32:64] = hi + w1 * torch.rand(32, generator=g) * 40
    z = (torch.randn(rows, n, generator=g) * 3)
    if rising:           # logits rising by 5e-4 per bar: a lane's running max moves by 1.6 % per step
        z = 5e-4 * torch.arange(n, dtype=F32).expand(rows, n) + 1e-3 * torch.randn(rows, n, generator=g)
    return z, y, borders


@pytest.mark.parametrize("n", [2, 33, 100, 1000])
def test_bar_restatement_inside_bound_at_c1(n):
    z, y, borders = _bar_data(512, n, n)
    f = EB.bar_nll_fwd(z, y, borders, True)
    lse = bar_lse(z)
    EB.check(f"host bar lse n={n}", lse, f["lse"], f["lse_bound"], 1.0)
    EB.check(f"host bar nll n={n}", bar_nll(z, y, borders, True, lse), f["nll"], f["nll_bound"], 1.0)
    g = torch.randn(512)
    k = f["idx"].clamp(0, n - 1)
    dl = (torch.exp(z - lse.unsqueeze(1)) - torch.zeros_like(z).scatter_(1, k.unsqueeze(1), 1.0)) * g.unsqueeze(1)
    exact, bound = EB.bar_nll_bwd(z, k, lse, g, EB.U32)
    EB.check(f"host bar dlogits n={n}", dl, exact, bound, 1.0)


def test_bar_neg_inf_first_bar_of_a_lane():
    """A -inf logit in a lane's first bar: expf(-inf - -inf) would make the row's lse NaN; log_softmax is finite."""
    z, y, borders = _bar_data(64, 100, 9)
    z[:, 5] = float("-inf")
    z[3] = float("-inf")
    ref = torch.logsumexp(z.double(), 1)
    assert torch.isnan(bar_lse(z, skip_neg_inf=False)[0])                 # the lane loop without the skip
    lse = bar_lse(z)
    ok = torch.arange(64) != 3
    f = EB.bar_nll_fwd(z, y, borders, False)
    EB.check("host bar lse with -inf", lse[ok], ref[ok], f["lse_bound"][ok], 1.0)
    assert lse[3].item() == float("-inf")


def test_bar_slips_outside_bound():
    # a half-normal constant off by 1e-5 (old: 1e-4 max|nll| + 1e-5)
    z, y, borders = _bar_data(2048, 100, 10)
    f = EB.bar_nll_fwd(z, y, borders, True)
    lse = bar_lse(z)
    got = bar_nll(z, y, borders, True, lse, half_log_2pi=HALF_LOG_2PI_F32 + 1e-5)
    r = _ratio(got, f["nll"], f["nll_bound"])
    old = (got.double() - f["nll"]).abs().max().item() <= 1e-4 * f["nll"].abs().max().item() + 1e-5
    _report("bar_nll half_log_2pi+1e-5", r, EB.C_BAR, old)
    assert r > EB.C_BAR and old
    # the online lse without the rescale when the running max rises by less than 2 %
    z, y, borders = _bar_data(256, 1000, 11, rising=True)
    f = EB.bar_nll_fwd(z, y, borders, True)
    lse = bar_lse(z, lazy=True)
    r = _ratio(lse, f["lse"], f["lse_bound"])
    got = bar_nll(z, y, borders, True, lse)
    old = (got.double() - f["nll"]).abs().max().item() <= 1e-4 * f["nll"].abs().max().item() + 1e-5
    _report("bar_nll lazy_rescale", r, EB.C_BAR, old)
    assert r > EB.C_BAR and not old
    # the backward's softmax formed from an lse off by 1e-6 (old: 1e-4 absolute)
    z, y, borders = _bar_data(2048, 100, 12)
    lse = bar_lse(z)
    k = EB.bucket_index(y, borders).clamp(0, 99)
    g = torch.randn(2048)
    dl = (torch.exp(z - (lse + 1e-6).unsqueeze(1)) - torch.zeros_like(z).scatter_(1, k.unsqueeze(1), 1.0)) * g.unsqueeze(1)
    exact, bound = EB.bar_nll_bwd(z, k, lse, g, EB.U32)
    r = _ratio(dl, exact, bound)
    old = (dl.double() - exact).abs().max().item() <= 1e-4
    _report("bar_nll_bwd lse+1e-6", r, EB.C_BAR_GRAD, old)
    assert r > EB.C_BAR_GRAD and old
    # a fast exponential (__expf: ex2.approx of fl32(x log2 e)); its argument's rounding alone, ex2 taken exact
    onehot = torch.zeros_like(z).scatter_(1, k.unsqueeze(1), 1.0)
    x = z - lse.unsqueeze(1)
    dl = (torch.exp2((x * torch.tensor(1.0 / math.log(2.0), dtype=F32)).double()).float() - onehot) * g.unsqueeze(1)
    r = _ratio(dl, exact, bound)
    old = (dl.double() - exact).abs().max().item() <= 1e-4
    _report("bar_nll_bwd fast exp", r, EB.C_BAR_GRAD, old)
    assert r > EB.C_BAR_GRAD and old


# ------------------------------------------------------------------------------------------------------------------
# Adam
# ------------------------------------------------------------------------------------------------------------------
def test_adam_helper_is_torch_adam_with_clip():
    """One step of the helper is clip_grad_norm_ + torch.optim.Adam (fp64 parameters, fp32-exact hyper-parameters)."""
    g = torch.Generator().manual_seed(13)
    lr, b1, b2, eps, wd = 0.0029296875, 0.875, 0.9990234375, 2.0 ** -27, 0.0078125     # exact in fp32
    p = torch.randn(300, generator=g, dtype=torch.float64)
    q = torch.nn.Parameter(p.clone())
    opt = torch.optim.Adam([q], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    m = torch.zeros(300, dtype=torch.float64)
    v = torch.zeros(300, dtype=torch.float64)
    for step in range(1, 6):
        grad = torch.randn(300, generator=g, dtype=torch.float64) * (5.0 if step % 2 else 1e-3)
        q.grad = grad.clone()
        norm_sq = (grad ** 2).sum().item()
        torch.nn.utils.clip_grad_norm_([q], 1.0)
        opt.step()
        ex = EB.adam_step(p, grad, m, v, step, lr, b1, b2, eps, wd, norm_sq, 1.0, 10)
        assert torch.allclose(ex["p"], q.detach(), rtol=0, atol=1e-13)
        assert torch.allclose(ex["m"], opt.state[q]["exp_avg"], rtol=0, atol=1e-13)
        assert torch.allclose(ex["v"], opt.state[q]["exp_avg_sq"], rtol=0, atol=1e-15)
        p, m, v = ex["p"], ex["m"], ex["v"]


def adam_f32(p, m, v, grad, step, clip, lr=1e-3, b1=0.9, b2=0.999, eps=1e-8):
    """adam_update_kernel's adam_one in fp32 with the kernel's clip coefficient."""
    n = p.numel()
    fb1, fb2 = torch.tensor(b1, dtype=F32), torch.tensor(b2, dtype=F32)
    bc1 = 1 - fb1 ** step
    bc2s = torch.sqrt(1 - fb2 ** step)
    gc = grad * torch.tensor(clip, dtype=F32)
    m = _fma(fb1.expand(n), m, (1 - fb1) * gc)
    v = _fma(fb2.expand(n), v, (1 - fb2) * gc * gc)
    p = p - (torch.tensor(lr, dtype=F32) / bc1) * (m / (torch.sqrt(v) / bc2s + torch.tensor(eps, dtype=F32)))
    return p, m, v


def test_adam_restatement_inside_bound_at_c1():
    g = torch.Generator().manual_seed(14)
    n = 5000
    p = torch.randn(n, generator=g)
    m = torch.zeros(n)
    v = torch.zeros(n)
    for step in range(1, 301):
        grad = torch.randn(n, generator=g) * (3.0 if step % 3 == 0 else 1e-3)
        norm_sq = (grad.double() ** 2).sum().item()
        ex = EB.adam_step(p, grad, m, v, step, 1e-3, 0.9, 0.999, 1e-8, 0.0, norm_sq, 1.0, EB.adam_norm_depth(1))
        clip = min(1.0, float(torch.tensor(1.0) / (torch.sqrt(torch.tensor(norm_sq, dtype=F32)) + 1e-6)))
        p, m, v = adam_f32(p, m, v, grad, step, clip)
        for key, got in (("p", p), ("m", m), ("v", v)):
            r = _ratio(got, ex[key], ex[key + "_bound"])
            assert r <= 1.0, (step, key, r)


def test_adam_clip_at_the_threshold_inside_bound_at_c1():
    """A gradient norm that puts the exact clip coefficient just above 1 while the kernel's fp32 norm, within its
    error, gives one just below 1: the kernel clips and the exact step does not, and the bound allows it."""
    g = torch.Generator().manual_seed(15)
    n = 5000
    grad = torch.randn(n, generator=g, dtype=torch.float64)
    grad = (grad / grad.norm() * (1.0 - 1e-6 - 1e-9)).float()          # exact coefficient 1 / (norm + 1e-6) ~ 1 + 1e-9
    norm_sq = (grad.double() ** 2).sum().item()
    assert 1.0 / (math.sqrt(norm_sq) + 1e-6) >= 1.0
    p, m, v = torch.randn(n, generator=g), torch.zeros(n), torch.zeros(n)
    depth = EB.adam_norm_depth(1)
    ex = EB.adam_step(p, grad, m, v, 1, 1e-3, 0.9, 0.999, 1e-8, 0.0, norm_sq, 1.0, depth)
    kernel_clip = 1.0 - 8 * EB.U32                                      # well inside the norm's U32 (depth / 2 + 6)
    for key, got in zip(("p", "m", "v"), adam_f32(p, m, v, grad, 1, kernel_clip)):
        assert _ratio(got, ex[key], ex[key + "_bound"]) <= 1.0, key
