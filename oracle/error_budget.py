"""Per-element error bounds for the bf16 / fp32 kernels -- TEST INFRASTRUCTURE ONLY.

Each helper computes the exact result in fp64 from the kernel's own (already rounded) inputs, together with a bound on
how far a correct kernel may be from it, element by element.  The bound is built from a *magnitude tensor* M, the same
contraction applied to absolute values, so that it is as tight in a row whose values are small as in the tensor's
largest row:

    |got - exact|  <=  c * bound,     bound = u M + E

u is the unit roundoff of the storage type (U = 2^-8 for bf16, U32 = 2^-24 for fp32), and E collects absolute terms
that are not a rounding of the result itself (the GELU approximant's error, an error the kernel inherits from an input
it was handed).  `check` prints the worst ratio |got - exact| / bound and asserts it is at most c; each test's c is
measured on the H100 (DESIGN.md section 4) and is at least twice the worst ratio seen there.

The helpers run on whatever device their inputs are on (the GPU tests keep the fp64 work on the GPU).
"""
import math

import torch

U = 2.0 ** -8       # bf16 unit roundoff (8-bit significand)
U32 = 2.0 ** -24    # fp32 unit roundoff
LSE_UNIT = 2.0 ** -20

# The tensor-core GELU epilogues (csrc/common.cuh, "Fast erf-GELU"): the approximant's own error and the hardware
# tanh.approx's (relative 2^-11 of tanh, i.e. 2^-12 of Phi)
GELU_ABS, GELU_GRAD_ABS, TANH_REL = 3.7e-5, 9.3e-5, 2.0 ** -12

# Constants c of the GPU tests: at least twice the worst ratio measured on an H100 80GB HBM3 (400 W and 700 W power limits)
# (DESIGN.md section 4 lists the ratios)
C_ATT_OUT = 3.2       # attention output, tensor-core and SIMT kernels (worst 1.54)
C_ATT_LSE = 0.3       # attention lse (worst 0.126)
C_ATT_GRAD = 5.0      # attention dQ, dK, dV and the dQ column sums (worst 2.46, dK)
C_GEMM = 2.0          # GEMM results and epilogues (worst 0.99)
# fp32 accumulation over K in units of U32 K |A||B| (the worst case of a sequential K-term sum), one constant per path.
# The wgmma GEMMs reach 0.014 of it (fp32 output, K = 192; 0.008 at K = 512, 5e-4 at K = 2560, 8e-5 at K = 12800); the
# SIMT GEMM 0.17 (K = 17..300, three k-splits reduced by fp32 atomics)
C_ACC_TC = 0.03
# The engine's wgmma weight gradients sum over tokens whose products share a sign, so their partial sums grow with K and
# the accumulator's rounding errors, which have one sign (as from truncation), do not cancel: they reach 0.066 of
# U32 K |A||B| (in-projection wgrad, K = 640 tokens), against 0.014 for zero-mean random operands
C_ACC_WGRAD = 0.15
C_ACC_SIMT = 0.35
# Row kernels (rowwise.cu, bar_nll.cu, optimizer.cu).  Their fp32 sums are bounded by the depth of the kernel's reduction
# tree (a sum whose longest path adds d terms is within U32 d sum|x| of the exact sum): a worst case that random data
# reaches a small fraction of, so C_ROWSUM is well below 1.  Where a result is stored in bf16 its rounding alone reaches
# a ratio of 1.
C_LN = 2.0            # LayerNorm h, mean, rstd (worst 0.996, bf16 h; fp32: h 0.40, mean 0.14, rstd 0.13)
C_LN_GRAD = 2.0       # LayerNorm dz, dgamma, dbeta, colsum_out (worst 0.996, bf16 dz; column sums 0.28)
C_ROWSUM = 0.3        # colsum and the embedding backward's column sums (worst 0.147)
C_EMBED = 2.0         # embedding forward (worst 0.996, bf16 out)
C_BAR = 1.1           # bar-NLL lse and nll (worst 0.521, nll; lse 0.330)
C_BAR_GRAD = 2.0      # bar-NLL dlogits (worst 0.996, bf16 dlogits; 0.487 fp32)
C_ADAM = 2.0          # Adam p, m, v and the squared gradient norm (worst 0.998, p; m 0.40, v 0.52, norm 0.040)
# GP sampler (gp_sampler.cu): L L^T - K against U32 (min(i, j) + 3) |L||L|^T + E_K, and y - L z against U32 (33 +
# ceil((r + 1) / 32)) |L||z| (the kernel's own L).  The factor's first rows meet its bound nearly term for term
# (L_00^2 = fl(os + fl(noise + jitter)) through one sqrtf), so its ratio approaches 1; the draw's long sums stay well below.
C_GP_FACTOR = 1.8     # worst 0.850 (T = 1000, F = 128, Matern-5/2, TR = 128)
C_GP_Y = 0.6          # worst 0.259 (cfg 2 at full size)
# Engine stages (tests/test_gpu_engine_stages.py).  The elementwise dropout stores in the activation dtype, so its
# rounding alone reaches 1; the ROWDOT sums and the fused v-third bias gradient are worst cases random data reach a
# small fraction of.
C_DROPOUT = 2.0       # dropout (+ residual), forward and backward masking (worst 0.996, bf16 out; fp32 0.968)
C_ROWDOT = 0.07       # GEMM ROWDOT epilogue, the attention backward's delta (worst 0.031, kernel test; engine 0.027)
C_BIAS_FUSED = 0.05   # in-projection bias gradient, v third formed as colsum(dz1) W_out (worst 0.024, cfg 3)


def check(name, got, exact, bound, c, verbose=True):
    """Assert |got - exact| <= c * bound elementwise; print (verbose) and return the worst ratio.  Where the bound is 0
    the kernel must be exact."""
    err = (got.double() - exact.double()).abs()
    bound = bound.double().expand_as(err)
    if (err[bound == 0] > 0).any():
        raise AssertionError(f"{name}: nonzero error where the bound is 0")
    ratio = (err / bound.clamp_min(1e-300)).masked_fill(bound == 0, 0.0)
    worst = ratio.max().item() if ratio.numel() else 0.0
    if verbose:
        print(f"[error-budget] {name}: worst err/bound = {worst:.4g} (c = {c})")
    if not math.isfinite(worst) or worst > c:
        idx = int(ratio.flatten().argmax())
        raise AssertionError(f"{name}: err/bound {worst:.4g} > {c} at flat index {idx} "
                             f"(got {got.flatten()[idx].item():.6g}, exact {exact.flatten()[idx].item():.6g}, "
                             f"bound {bound.flatten()[idx].item():.3g})")
    return worst


# ------------------------------------------------------------------------------------------------------------------
# masked attention (keys(i) = [0, sep) U {i if i >= sep}), token-major [T*B, 3E] qkv with token = t*B + b
# ------------------------------------------------------------------------------------------------------------------
def _heads(t, T, B, H, dh):
    return t.reshape(T, B, H, dh).permute(1, 2, 0, 3)          # [B, H, T, dh]


def _tokens(t, T, B, H, dh):
    return t.permute(2, 0, 1, 3).reshape(T * B, H * dh)


def allowed_keys(T, sep, device):
    i = torch.arange(T, device=device).unsqueeze(1)
    j = torch.arange(T, device=device).unsqueeze(0)
    return (j < sep) | (i == j)


def attention_fwd(qkv, T, B, H, dh, sep, u, keep=None, drop_scale=1.0):
    """Exact forward and its bounds.  keep: optional 0/1 dropout mask [B, H, T, T] on the probabilities (kept entries
    scaled by drop_scale).

    out: the kernel rounds P (<= 1) and O / l to the storage type, each a relative error u: u * P^|V| with
    P^ = softmax * keep * drop_scale.  The fp32 scores carry an error of order U32 a_i, a_i = 1 + scale max_j
    sum_d |q_id k_jd|, which moves every probability of the row by that relative amount: the unit is u + U32 a_i.
    lse (fp32): LSE_UNIT (1 + |lse| + a_i)."""
    E = H * dh
    x = qkv.double()
    q, k, v = (_heads(x[:, n * E:(n + 1) * E], T, B, H, dh) for n in range(3))
    scale = 1.0 / math.sqrt(dh)
    ok = allowed_keys(T, sep, x.device)
    s = (q @ k.transpose(-1, -2) * scale).masked_fill(~ok, float("-inf"))
    lse = torch.logsumexp(s, -1)
    P = torch.exp(s - lse.unsqueeze(-1))
    Ph = P if keep is None else P * keep.double() * drop_scale
    a = 1.0 + ((q.abs() @ k.abs().transpose(-1, -2)) * scale).masked_fill(~ok, 0.0).amax(-1)   # [B, H, T]
    unit = u + U32 * a
    out = Ph @ v
    out_bound = unit.unsqueeze(-1) * (Ph @ v.abs())
    return {"T": T, "B": B, "H": H, "dh": dh, "u": u, "scale": scale, "q": q, "k": k, "v": v, "P": P, "Ph": Ph,
            "keep": keep, "drop_scale": drop_scale, "unit": unit,
            "out": _tokens(out, T, B, H, dh), "out_bound": _tokens(out_bound, T, B, H, dh),
            "lse": lse.reshape(B * H, T), "lse_bound": (LSE_UNIT * (1.0 + lse.abs() + a)).reshape(B * H, T)}


def rising_max_qkv(T, B, H, dh, generator=None, device=None):
    """Data on which the running max of the online softmax moves by less than 2 % per 64-key block: q along e0 and every
    key of block kb at 1 + 3/128 kb along e0 (exact in bf16), so the block maxima rise by 0.017 (corr = 0.983); v has a
    mean offset so that the output does not cancel and a skipped rescale of O shows."""
    E = H * dh
    x = torch.zeros(T, B, 3, H, dh, dtype=torch.float64)
    x[:, :, 0, :, 0] = 8.0
    x[:, :, 1, :, 0] = (1.0 + 3.0 / 128.0 * (torch.arange(T, dtype=torch.float64) // 64)).view(T, 1, 1)
    x[:, :, 1, :, 1:] = 0.01 * torch.randn(T, B, H, dh - 1, generator=generator, dtype=torch.float64)
    x[:, :, 2] = 1.0 + torch.randn(T, B, H, dh, generator=generator, dtype=torch.float64)
    return x.reshape(T * B, 3 * E).to(device=device, dtype=torch.bfloat16)


def attention_bwd(f, dout, out_kernel, delta_kernel=None):
    """Exact dQ, dK, dV (token-major [T*B, E] each) of the forward `f` for the upstream gradient dout, and their bounds.

    dS = P (dP - delta) with dP = keep drop_scale dO V^T and delta_i = dO_i . out_i.  The kernel rounds P and dS to the
    storage type before the second MMAs and the results at the end, so with |dS|~ = P (|dP| + |delta|):
      dV: unit P^^T |dO|
      dQ: scale (unit |dS|~ |K| + e_delta P |K|)
      dK: scale (|dS|~^T (unit |Q|) + P^T (e_delta |Q|))
    where e_delta,i = |dO_i . (out_kernel - out_exact)_i| is the error the kernel inherits by forming delta from the
    output it stored (not a rounding of its own, so it is not scaled by u).  delta_kernel: a token-major [T*B, H] delta
    handed to the kernel precomputed (the GEMM ROWDOT epilogue); its own deviation |delta_kernel - dO . out_kernel| from
    the delta of the stored output adds to e_delta."""
    T, B, H, dh = f["T"], f["B"], f["H"], f["dh"]
    scale, P, Ph, q, k, v = f["scale"], f["P"], f["Ph"], f["q"], f["k"], f["v"]
    unit = f["unit"].unsqueeze(-1)
    do = _heads(dout.double(), T, B, H, dh)
    out = _heads(f["out"], T, B, H, dh)
    dPh = do @ v.transpose(-1, -2)
    dP = dPh if f["keep"] is None else dPh * f["keep"].double() * f["drop_scale"]
    delta = (do * out).sum(-1, keepdim=True)
    dS = P * (dP - delta)
    dS_mag = P * (dP.abs() + delta.abs())
    out_k = _heads(out_kernel.double(), T, B, H, dh)
    e_delta = (do * (out_k - out)).sum(-1, keepdim=True).abs()
    if delta_kernel is not None:
        dk_ = delta_kernel.double().reshape(T, B, H).permute(1, 2, 0).unsqueeze(-1)
        e_delta = e_delta + (dk_ - (do * out_k).sum(-1, keepdim=True)).abs()
    dq = scale * (dS @ k)
    dk = scale * (dS.transpose(-1, -2) @ q)
    dv = Ph.transpose(-1, -2) @ do
    dq_b = scale * (unit * (dS_mag @ k.abs()) + e_delta * (P @ k.abs()))
    dk_b = scale * ((unit * dS_mag).transpose(-1, -2) @ q.abs() + P.transpose(-1, -2) @ (e_delta * q.abs()))
    dv_b = (unit * Ph).transpose(-1, -2) @ do.abs()
    tok = lambda t: _tokens(t, T, B, H, dh)
    return {"dq": tok(dq), "dk": tok(dk), "dv": tok(dv), "dq_bound": tok(dq_b), "dk_bound": tok(dk_b), "dv_bound": tok(dv_b)}


def check_attention_fwd(out, lse, f, c_out, c_lse, tag=""):
    """Both outputs of the forward against `f` = attention_fwd(...)."""
    r_out = check(f"attention out{tag}", out, f["out"], f["out_bound"], c_out)
    r_lse = check(f"attention lse{tag}", lse, f["lse"], f["lse_bound"], c_lse)
    return r_out, r_lse


def check_attention_bwd(dqkv, b, c, tag=""):
    """dqkv [T*B, 3E] against `b` = attention_bwd(...); returns the worst ratio over dq, dk, dv."""
    E = b["dq"].shape[1]
    return max(check(f"attention {name}{tag}", dqkv[:, n * E:(n + 1) * E], b[name], b[name + "_bound"], c)
               for n, name in enumerate(("dq", "dk", "dv")))


# ------------------------------------------------------------------------------------------------------------------
# GEMM  C = epi(A B^T + bias) (+ aux), A [M, K], B [N, K] as logical (already transposed) operands
# ------------------------------------------------------------------------------------------------------------------
def gemm(A, B, u_out, c_acc, bias=None, aux=None, epilogue="none", fast_gelu=True):
    """Exact result and bound of one GEMM launch.  A, B: the logical [M, K] / [N, K] operands (bf16 or fp32 values).

    The fp32 accumulation over K contributes c_acc U32 K (|A||B|^T) -- the worst-case model of a K-term sum, scaled by the
    constant measured for the kernel's path (C_ACC_TC, C_ACC_SIMT) -- and storing the result u_out times the magnitude of each term the epilogue
    adds.  epilogue:
      "none"      acc + bias (+ aux)
      "gelu"      gelu(acc + bias) (+ aux), with the fast-GELU approximant's error (GELU_ABS + TANH_REL |x|)
      "gelu_grad" gelu'(acc + bias), the forward's C2 output (GELU_GRAD_ABS + TANH_REL (1 + |x|))
      "gelu_bwd"  acc * gelu'(aux)
      "mul"       acc * aux
    fast_gelu=False for the SIMT kernels, which evaluate erff: no approximant term.  Returns (exact, bound, pre) with pre = acc + bias in fp64."""
    Ad, Bd = A.double(), B.double()
    K = Ad.shape[1]
    acc = Ad @ Bd.t()
    acc_err = c_acc * U32 * K * (Ad.abs() @ Bd.abs().t())
    pre = acc if bias is None else acc + bias.double()
    g_abs, g_grad_abs, t_rel = (GELU_ABS, GELU_GRAD_ABS, TANH_REL) if fast_gelu else (0.0, 0.0, 0.0)
    auxd = None if aux is None else aux.double()
    if epilogue in ("none", "gelu"):
        if epilogue == "gelu":
            cdf = 0.5 * (1.0 + torch.erf(pre / math.sqrt(2.0)))
            val = pre * cdf
            bound = u_out * val.abs() + 1.13 * acc_err + g_abs + t_rel * pre.abs()
        else:
            val = pre
            bound = u_out * pre.abs() + acc_err
        if auxd is not None:
            val = val + auxd
            bound = bound + u_out * auxd.abs()
        return val, bound, pre
    if epilogue == "gelu_grad":
        val = gelu_grad(pre)
        return val, u_out * val.abs() + 1.13 * acc_err + g_grad_abs + t_rel * (1.0 + pre.abs()), pre
    if epilogue == "gelu_bwd":
        gp = gelu_grad(auxd)
        val = acc * gp
        bound = u_out * val.abs() + acc_err * gp.abs() + acc.abs() * (g_grad_abs + t_rel * (1.0 + auxd.abs()))
        if not fast_gelu:
            # erff / __expf evaluate Phi and x phi(x) to a few U32 each (__expf: 2 + 1.16 |arg| ulp) and the two terms
            # cancel for x < 0: gelu' is good to U32 times the terms' magnitude, not its own (measured 25x over U32 |gelu'|)
            ax = auxd.abs()
            bound = bound + acc.abs() * U32 * (2.0 + ax * torch.exp(-0.5 * ax * ax) / math.sqrt(2.0 * math.pi) * (6.0 + ax + 2.0 * ax * ax))
        return val, bound, pre
    if epilogue == "mul":
        val = acc * auxd
        return val, u_out * val.abs() + acc_err * auxd.abs(), pre
    raise ValueError(epilogue)


def gelu_grad(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


# ------------------------------------------------------------------------------------------------------------------
# Row kernels: LayerNorm, embedding, column sums (csrc/rowwise.cu), bar NLL (csrc/bar_nll.cu), Adam (csrc/optimizer.cu).
# Their fp32 sums are bounded by the depth of the kernel's reduction tree: a sum formed as a tree whose longest
# root-to-leaf path has d additions is within U32 d sum|x| of the exact sum, whatever the order.  The launch geometry
# that sets the depth is passed in (num_sms), so that the host test evaluates the same bounds without a device.
# ------------------------------------------------------------------------------------------------------------------
def _cdiv(a, b):
    return -(-a // b)


def ln_lane_depth(E):
    """Additions on the longest path of a LayerNorm row sum: a lane's serial sum (8 elements per 256-column chunk on
    the vector path, ceil(E / 32) on the generic one), the 5-level warp butterfly and the scaling by 1 / E."""
    return max(8 * _cdiv(E, 256), _cdiv(E, 32)) + 5 + 2


def ln_vec(E, ld_list, ptrs_aligned=True):
    """Whether the LayerNorm launch takes the vector kernel (rowwise.cu layernorm_*_dispatch)."""
    return E % 8 == 0 and E <= 1024 and all(ld % 8 == 0 for ld in ld_list) and ptrs_aligned


def ln_bwd_colsum_depth(rows, E, elem_size, vec, num_sms):
    """Depth of the backward's column sums (dgamma, dbeta, colsum_out) over rows, plus the initial value of the output.
    Vector kernel: a lane's serial sum over the rows its warp owns, 8 warps into shared memory, one global atomic per
    CTA.  Generic kernel: one global atomic per row."""
    if not vec:
        return rows + 1
    row_bytes = 256 * _cdiv(E, 256) * elem_size
    ctas = 2 if row_bytes <= 512 else 1
    grid = min(ctas * num_sms, _cdiv(rows, 8))
    return _cdiv(rows, grid * 8) + 8 + grid + 1


def layernorm_fwd(z, gamma, beta, u, eps=1e-5):
    """Exact h, mean, rstd of LayerNorm over the last dim, and their bounds.

    mean: U32 a_mu mean|z| with a_mu the row sum's depth.  The variance is summed about the kernel's mean: each term
    rounds twice (z - mu, the fma), the sum has the same depth, and the mean's error adds (mu^ - mu)^2; rsqrtf and
    the + eps add a few more, so rstd is within U32 (a_r + 4) + (mu^ - mu)^2 / (2 (var + eps)) of r relatively.
    h: u |h| + U32 (|gamma| r (|z - mu| a_r + a_mu mean|z|) + |beta|)."""
    zd, gd, bd = z.double(), gamma.double(), beta.double()
    E = zd.shape[-1]
    mu = zd.mean(-1, keepdim=True)
    var = ((zd - mu) ** 2).mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt(var + eps)
    h = (zd - mu) * r * gd + bd
    a = ln_lane_depth(E)
    mabs = zd.abs().mean(-1, keepdim=True)
    mu_b = U32 * a * mabs
    r_rel = U32 * (a + 4) + 0.5 * mu_b ** 2 / (var + eps)
    h_b = u * h.abs() + U32 * (gd.abs() * r * ((zd - mu).abs() * (a + 4) + a * mabs) + bd.abs()) + gd.abs() * (zd - mu).abs() * r * r_rel
    return {"h": h, "h_bound": h_b, "mean": mu.squeeze(-1), "mean_bound": mu_b.squeeze(-1),
            "rstd": r.squeeze(-1), "rstd_bound": (r * r_rel).squeeze(-1)}


def layernorm_bwd(dh, z, gamma, mean_k, rstd_k, u, colsum_depth, init=None, eps=1e-5):
    """Exact dz, dgamma, dbeta, colsum_out = sum_rows dz of LayerNorm for the upstream dh, and their bounds.

    The exact values use fp64 statistics of z.  The kernel reads the mean and rstd the forward stored (mean_k, rstd_k);
    their actual deviation from the exact ones moves x^ = (z - mu) r by e_x = r |mu^ - mu| + |x^| |r^ / r - 1|, an
    inherited term E.  dz = r (g - mean g - x^ mean(g x^)), g = dh gamma: the three terms cancel, so its rounding is
    bounded by their magnitudes, U32 (a + 4) r (|g| + mean|g| + |x^| mean|g x^|) with a the row sum's depth, plus
    u |dz| for the store.  The column sums over rows: U32 colsum_depth times the sum of the terms' magnitudes.
    init: the values the column outputs held before the call (accumulated into); eps: the forward's."""
    zd, dd, gd = z.double(), dh.double(), gamma.double()
    E = zd.shape[-1]
    mu = zd.mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt(((zd - mu) ** 2).mean(-1, keepdim=True) + eps)
    xh = (zd - mu) * r
    g = dd * gd
    s1, s2 = g.mean(-1, keepdim=True), (g * xh).mean(-1, keepdim=True)
    dz = r * (g - s1 - xh * s2)
    a = ln_lane_depth(E)
    eps_r = (rstd_k.double().view_as(r) / r - 1.0).abs()
    e_x = (r * (mean_k.double().view_as(mu) - mu).abs() + xh.abs() * eps_r) * (1.0 + 4 * U32)   # (z - mu^) r^ rounds too
    dz_mag = r * (g.abs() + g.abs().mean(-1, keepdim=True) + xh.abs() * (g * xh).abs().mean(-1, keepdim=True))
    dz_inh = eps_r * dz.abs() + r * (e_x * s2.abs() + xh.abs() * (g.abs() * e_x).mean(-1, keepdim=True))
    dz_b = u * dz.abs() + U32 * (a + 4) * dz_mag + dz_inh
    if init is None:
        init = torch.zeros(3, E, dtype=torch.float64, device=zd.device)
    init = [t.double() for t in init]
    d_col = U32 * (colsum_depth + 3)
    out = {"dz": dz, "dz_bound": dz_b,
           "dgamma": init[0] + (dd * xh).sum(0),
           "dgamma_bound": d_col * ((dd * xh).abs().sum(0) + init[0].abs()) + (dd.abs() * e_x).sum(0),
           "dbeta": init[1] + dd.sum(0),
           "dbeta_bound": d_col * (dd.abs().sum(0) + init[1].abs()),
           "colsum": init[2] + dz.sum(0),
           # colsum_out sums the kernel's fp32 dz before it is stored: its terms carry dz's fp32 error, not the store's
           "colsum_bound": d_col * (dz.abs().sum(0) + init[2].abs()) + (dz_b - u * dz.abs() + U32 * dz.abs()).sum(0)}
    return out


def colsum_depth(rows, N, ld, elem_size, num_sms, aligned=True):
    """Depth of pfn_colsum's column sums (rowwise.cu colsum_dispatch), plus the initial value of out."""
    if N % 8 == 0 and ld % 8 == 0 and aligned:
        gx = min(num_sms * 4, _cdiv(rows, 8))
        if N <= 512:
            grid = gx
        else:
            groups = _cdiv(N, 1024)
            grid = min((gx * 2) // groups if gx // groups > 0 else 1, _cdiv(rows, 8))
        return _cdiv(rows, grid * 8) + 8 + grid + 1
    rows_per_cta = max(64, _cdiv(rows, num_sms * 2))
    return rows_per_cta + _cdiv(rows, rows_per_cta) + 1


def colsum(X, init, depth, block_rows=1 << 16):
    """Exact init + X.sum(0) and its bound U32 depth (sum|X| + |init|).  The fp64 sums run over blocks of rows, so that
    a full-size X needs no fp64 copy of itself."""
    s, a = init.double().clone(), init.double().abs()
    for r0 in range(0, X.shape[0], block_rows):
        Xd = X[r0:r0 + block_rows].double()
        s += Xd.sum(0)
        a += Xd.abs().sum(0)
    return s, U32 * depth * a


def dropout(x, keep, thr, residual=None, u_out=U):
    """Exact x keep s (+ residual) of the elementwise dropout kernel (dropout.cu), s = 256 / (256 - thr) in fp64: the
    kernel's contract is probability thr / 256 at that scale (not the reference's p).  The kernel multiplies by
    fl32(s) and rounds in fp32, adds the residual in fp32 and stores: |fl32(s) - s| |x| keep + U32 (|x| s keep + |val|)
    + u_out |val|."""
    xd, kd = x.double(), keep.double()
    s = 256.0 / (256.0 - thr)
    s32 = _f32(s)
    kept = xd.abs() * kd
    val = xd * kd * s
    if residual is not None:
        val = val + residual.double()
    return val, u_out * val.abs() + U32 * (kept * s + val.abs()) + abs(s32 - s) * kept


def rowdot_depth(width, block_n=128):
    """Longest addition chain of a ROWDOT sum (gemm_tc.cu epi_pair / the epilogue's quad shuffles): a lane's fmaf chain
    over its block_n / 4 columns of one tile, two shuffles, one atomic per tile of the group, the zeroed initial value."""
    return block_n // 4 + 2 + _cdiv(width, block_n) + 1


def rowdot(C, aux, width):
    """Exact sum over each group of `width` columns of C aux, with C the GEMM's stored (bf16) output, and its bound
    U32 depth sum |C aux| (the products of two bf16 values are exact in fp32; only the additions round).  A last
    group narrower than width sums the columns that exist."""
    M, N = C.shape
    prod = C.double() * aux.double()
    groups = _cdiv(N, width)
    pad = groups * width - N
    if pad:
        prod = torch.nn.functional.pad(prod, (0, pad))
    prod = prod.view(M, groups, width)
    return prod.sum(-1), U32 * rowdot_depth(width) * prod.abs().sum(-1)


def bias_v_fused(dattn, da, out_w, colsum_out, ln_b, c_acc):
    """Bound of the in-projection bias gradient's v third when it is formed as colsum_out W_out (fp32) instead of the
    column sums of dV.  The exact value is sum_i dO_i over the stored dO = dattn (the rows of P sum to 1), so the bound
    collects how far colsum_out W_out may be from it:
      U sum_i |dattn_i| + c_acc U32 E sum_i |da_i| |W_bf16|   the bf16 rounding and fp32 accumulation of the dgrad
      U |colsum_out| |W|                                      the dgrad read bf16(W), the product reads the fp32 master
      (colsum_bound + sum_i dz_bound_i) |W|                   colsum_out (the LayerNorm backward's fp32 sums of dz)
                                                              against the column sums of the stored dz = da
      U32 E |colsum_out| |W|                                  the fp32 matrix-vector product
    with W = out_w [E_out, E_in] (fp32 master) and ln_b the layernorm_bwd bounds of that LayerNorm."""
    W = out_w.double()
    Wa = W.abs()
    Wb = out_w.to(torch.bfloat16).double().abs()
    E = W.shape[0]
    cs = colsum_out.double().abs()
    inh = ln_b["colsum_bound"] + ln_b["dz_bound"].sum(0)
    return (U * dattn.double().abs().sum(0) + c_acc * U32 * E * (da.double().abs().sum(0) @ Wb)
            + (U * cs + inh + U32 * E * cs) @ Wa)


def embed_fwd(x, y, Wx, bx, wy, by, sep, u):
    """Exact embedding x Wx^T + bx (+ y wy + by on the first sep*B rows), x [rows, F], and its bound
    u |out| + U32 (F + 2) (|x||Wx|^T + |bx| + |y wy| + |by|)."""
    xd, yd = x.double(), y.double().reshape(-1, 1)
    W, b, w, bb = Wx.double(), bx.double(), wy.double().reshape(1, -1), by.double()
    train = (torch.arange(xd.shape[0], device=xd.device) < sep).double().unsqueeze(1)
    out = xd @ W.t() + b + train * (yd * w + bb)
    mag = xd.abs() @ W.abs().t() + b.abs() + train * ((yd * w).abs() + bb.abs())
    return out, u * out.abs() + U32 * (W.shape[1] + 2) * mag


def embed_bwd_depth(rows):
    """embed_bwd: a thread sums its column over a CTA's 512 rows, then one global atomic per CTA, plus the initial value."""
    return min(rows, 512) + _cdiv(rows, 512) + 1


def embed_bwd(dout, x, y, sep, depth):
    """Exact dWx, dbx, dwy, dby of the embedding for dout [rows, E] (train rows: the first sep*B), and their bounds."""
    dd, xd, yd = dout.double(), x.double(), y.double().reshape(-1)
    t = (torch.arange(dd.shape[0], device=dd.device) < sep).double()
    d_col = U32 * (depth + 1)
    return {"dWx": (dd.t() @ xd, d_col * (dd.abs().t() @ xd.abs())),
            "dbx": (dd.sum(0), d_col * dd.abs().sum(0)),
            "dwy": ((t * yd) @ dd, d_col * ((t * yd).abs() @ dd.abs())),
            "dby": (t @ dd, d_col * (t @ dd.abs()))}


# bar NLL -----------------------------------------------------------------------------------------------------------
ICDF_HALF = 0.6744897501960817
HALF_LOG_2PI = 0.5 * math.log(2.0 * math.pi)


def bucket_index(y, borders):
    """searchsorted-left minus one with the edge fix-ups (bar_distribution.py:19-23), on the inputs' device."""
    b = borders.double()
    yd = y.double()
    idx = torch.searchsorted(b, yd) - 1
    idx = torch.where(yd == b[0], torch.zeros_like(idx), idx)
    return torch.where(yd == b[-1], torch.full_like(idx, b.numel() - 2), idx)


def bar_nll_fwd(logits, y, borders, full_support):
    """Exact lse and nll of the bar distribution (log_softmax over the bars, so -inf logits add nothing), and bounds.

    lse: U32 (|lse| + A + ceil(n / 32) + 12), A the row's largest |z - lse| over finite logits: each exp term carries
    U32 |z - m| from its rounded argument, a lane sums ceil(n / 32) terms, the warp combine and logf a few more.
    nll: U32 (|z_k| + |lse| + 2 |log w| + 4) plus the lse bound.  The width w = b[k+1] - b[k] and the tails' distance
    v = b[1] - y / y - b[n-1] are differences of the kernel's fp32 inputs, so fp32 rounds each to within U32 of itself
    (e_w = e_v = U32) however narrow the bucket is next to its borders.  The tails add U32 (|log s| + 2 + 6 t) +
    2 t (e_v + e_w) with t = v^2 / (2 s^2) the half-normal's quadratic term."""
    z = logits.double()
    n = z.shape[-1]
    b = borders.double()
    yd = y.double()
    lse = torch.logsumexp(z, -1)
    fin = torch.isfinite(z)
    A = torch.where(fin, (z - lse.unsqueeze(-1)).abs(), torch.zeros_like(z)).amax(-1)
    lse_b = U32 * (lse.abs() + A + _cdiv(n, 32) + 12)
    idx = bucket_index(y, borders)
    if full_support:
        idx = idx.clamp(0, n - 1)
    k = idx.clamp(0, n - 1)
    w = (b[1:] - b[:-1])[k]
    e_w = U32
    zk = z.gather(-1, k.unsqueeze(-1)).squeeze(-1)
    logp = zk - lse - torch.log(w)
    bound = U32 * (zk.abs() + lse.abs() + 2.0 * torch.log(w).abs() + 4) + lse_b + e_w
    if full_support:
        for side in (0, n - 1):
            sel = k == side
            v = (b[1] - yd).clamp_min(1e-8) if side == 0 else yd - b[n - 1]
            e_v = U32
            wb = b[side + 1] - b[side]
            s = wb / ICDF_HALF
            t = v * v / (2.0 * s * s)
            hn = math.log(2.0) - torch.log(s) - HALF_LOG_2PI - t
            logp = torch.where(sel, logp + hn + torch.log(wb), logp)
            tb = U32 * (torch.log(s).abs() + 2 + 6 * t) + 2 * t * (e_v + e_w) + e_w
            bound = torch.where(sel, bound + tb, bound)
    oob = (idx < 0) | (idx >= n)
    nll = torch.where(oob, torch.full_like(logp, float("nan")), -logp)
    return {"lse": lse, "lse_bound": lse_b, "nll": nll, "nll_bound": bound, "idx": idx}


def bar_nll_bwd(logits, idx, lse, g, u_d):
    """Exact dlogits = g (exp(x) - onehot(idx)) and its bound, with x = fl32(z - lse) the kernel's own fp32 argument
    (formed from the lse the forward stored; an IEEE fp32 subtraction, so the device forms the same x).  Taking x as
    the kernel's input leaves only expf's documented 2 ulp (4 U32 relative), the - 1, the * g and the store:
    u_d |dl| + U32 |g| (4 p + |p - [c = k]|) + U32 |dl|, relative to each probability, so the small ones are bounded
    too.  A fast exponential (ex2.approx of x log2 e) adds about U32 |x|, which this bound does not allow."""
    x = (logits.float() - lse.float().unsqueeze(-1)).double()
    gd = g.double().unsqueeze(-1)
    p = torch.exp(x)
    onehot = torch.zeros_like(p).scatter_(-1, idx.unsqueeze(-1), 1.0)
    dl = gd * (p - onehot)
    return dl, (u_d + U32) * dl.abs() + U32 * gd.abs() * (4 * p + (p - onehot).abs())


# Adam ---------------------------------------------------------------------------------------------------------------
def adam_norm_depth(n_chunks):
    """Depth of the squared-gradient-norm sum: a thread's serial sum over its share of an 8192-element chunk (32 on the
    scalar path, 8 float4 of four products on the vector one), the warp and CTA butterflies, one atomic per chunk."""
    return 32 + 4 + 8 + n_chunks + 2


def adam_step(p, g, m, v, step, lr, beta1, beta2, eps, weight_decay, clip_norm_sq, max_grad_norm, norm_depth):
    """Exact fp64 result of one torch.optim.Adam step (after clip_grad_norm_) from the state before it (p, m, v: the
    kernel's own fp32 values), and bounds.  The hyper-parameters are taken as the kernel's fp32 values.

    clip_norm_sq: exact sum of g^2 over every tensor of the step; the kernel's fp32 norm carries U32 norm_depth
    relative, so the clip coefficient carries half of it plus a few roundings (e_c).  Within that error of 1 the
    kernel may clip where the exact coefficient does not, or not clip where it does; e_c covers both.  m: 3 U32 (|b1 m| + |(1-b1) g'|) +
    (1-b1)|g'| e_c; v likewise.  p: the update's error through m, v and the bias corrections (powf and 1 - b^t:
    U32 (3 b^t / (1 - b^t) + 2)), then U32 |p_new|."""
    f = lambda x: float(torch.tensor(x, dtype=torch.float32))
    lr, beta1, beta2, eps, wd = f(lr), f(beta1), f(beta2), f(eps), f(weight_decay)
    pd, gd, md, vd = p.double(), g.double(), m.double(), v.double()
    e_c = 0.0
    clip = 1.0
    if max_grad_norm and max_grad_norm > 0:
        norm = math.sqrt(clip_norm_sq)
        c = f(max_grad_norm) / (norm + 1e-6)
        e_norm = U32 * (0.5 * norm_depth + 6)
        if c < 1.0 + 2 * e_norm:
            clip = min(c, 1.0)
            e_c = e_norm
    gp = gd * clip
    gp_b = gp.abs() * (e_c + U32)
    if wd != 0.0:
        gp = gp + wd * pd
        gp_b = gp_b + U32 * (wd * pd.abs() + gp.abs())
    m1 = beta1 * md + (1 - beta1) * gp
    m_b = 3 * U32 * (beta1 * md.abs() + (1 - beta1) * gp.abs()) + (1 - beta1) * gp_b
    v1 = beta2 * vd + (1 - beta2) * gp * gp
    v_b = 4 * U32 * v1 + (1 - beta2) * 2 * gp.abs() * gp_b
    bc1 = 1 - beta1 ** step
    bc2s = math.sqrt(1 - beta2 ** step)
    e_bc1 = U32 * (3 * beta1 ** step / bc1 + 2)
    e_bc2 = U32 * (3 * beta2 ** step / (1 - beta2 ** step) + 2)
    sq = torch.sqrt(v1) / bc2s
    denom = sq + eps
    step_size = lr / bc1
    delta = step_size * m1 / denom
    rel_v = v_b / v1.clamp_min(1e-300)
    delta_b = step_size / denom * m_b + delta.abs() * (0.5 * (rel_v + e_bc2) * sq / denom + e_bc1 + 6 * U32)
    p1 = pd - delta
    return {"p": p1, "p_bound": U32 * p1.abs() + delta_b, "m": m1, "m_bound": m_b + U32 * m1.abs(),
            "v": v1, "v_bound": v_b}


# ------------------------------------------------------------------------------------------------------------------
# GP prior sampler (csrc/gp_sampler.cu): K = os k(x, x; ls) + (noise + jitter) I evaluated in fp32, its left-looking
# blocked fp32 Cholesky L (panel width 32) and y = L z.  Kernel types as in _lib.KERNEL_*.
# ------------------------------------------------------------------------------------------------------------------
GP_RBF, GP_MATERN12, GP_MATERN32, GP_MATERN52 = 0, 1, 2, 3
GP_PANEL = 32


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _is_f32(t):
    return t.float().double() == t


def _exact_add(a, b):
    """The fp64 sum or difference of two fp32 values is exact when their magnitudes lie within 2^28 of each other."""
    aa, bb = a.abs(), b.abs()
    return (aa == 0) | (bb == 0) | ((aa <= bb * 2.0 ** 28) & (bb <= aa * 2.0 ** 28))


def gp_kernel(x, ls, os_, noise, jitter, kernel_type):
    """Exact K + jitter I [B, T, T] from the kernel's fp32 inputs (x [B, T, F], ls [B, F], os_ [B], noise [B], jitter as
    the fp32 value the kernel receives), and an elementwise bound E_K on the kernel's fp32 evaluation of it.

    gp_kernel_value and its caller round il = 1/ls, x il (each relative U32), their difference, and d2 through an F-term
    fmaf chain.  Per feature s = (x_r - x_c) il is formed with error U32 (2|s| + a), a = (|x_r| + |x_c|) il: where the two
    products nearly cancel it is relative to a, not to s.  So d2 is within
        E_d2 = U32 ((F + 4) d2 + 2 sum_f |s_f| a_f) + U32^2 sum_f (2|s_f| + a_f)^2.
    The Matern kernels take r = sqrtf(d2): r moves by at most min(sqrt(E_d2), E_d2 / (sqrt(d2) + sqrt(d2 - E_d2))) plus
    sqrtf's own U32 r.  The rounded constants (sqrt 3, sqrt 5, 5/3 in fp32) move a = c r and the polynomial; each
    is carried into k by k's derivative.  expf is good to 2 ulp (4 U32 relative), and the products with os and the
    polynomial round once each.  Where expf's result is subnormal its error is absolute: (2 os p + 1/2) 2^-149.
    The diagonal is fl(os + fl(noise + jitter))."""
    xd, ld = x.double(), ls.double()
    B, T, F = xd.shape
    jit = _f32(jitter)
    d2 = torch.zeros(B, T, T, dtype=torch.float64, device=xd.device)
    s1 = torch.zeros_like(d2)
    s2 = torch.zeros_like(d2)
    # Where every intermediate of d2 (il, x il, the difference, its square, each partial sum) is an fp32 value and each
    # fp64 step forming it is exact, every fp32 rounding of the kernel is exact too, in whatever order or fusion: d2 has
    # no error there (dyadic x and lengthscales), which leaves expf and the constants alone in the bound
    exact = torch.ones(B, T, T, dtype=torch.bool, device=xd.device)
    acc = torch.zeros_like(d2)
    for f in range(F):
        il = (1.0 / ld[:, f]).view(B, 1, 1)
        ilf = (1.0 / ls[:, f].float()).double()
        xf = xd[:, :, f]
        s = (xf.unsqueeze(2) - xf.unsqueeze(1)) * il
        a = (xf.abs().unsqueeze(2) + xf.abs().unsqueeze(1)) * il
        d2 += s * s
        s1 += s.abs() * a
        s2 += (2.0 * s.abs() + a) ** 2
        xi = xf * ilf.view(B, 1)
        ok = (ilf * ld[:, f] == 1.0).view(B, 1) & _is_f32(xi)
        sf = xi.unsqueeze(2) - xi.unsqueeze(1)
        sq = sf * sf
        nxt = acc + sq
        exact &= (ok.unsqueeze(2) & ok.unsqueeze(1) & _exact_add(xi.unsqueeze(2), xi.unsqueeze(1)) & _is_f32(sf)
                  & _is_f32(sq) & _exact_add(acc, sq) & _is_f32(nxt))
        acc = nxt
    e_d2 = (U32 * ((F + 4) * d2 + 2.0 * s1) + U32 * U32 * s2).masked_fill(exact, 0.0)
    del s1, s2, acc, exact
    osv = os_.double().view(B, 1, 1)
    if kernel_type == GP_RBF:
        k = torch.exp(-0.5 * d2)
        poly = torch.ones_like(d2)
        e_k = k * (torch.expm1(0.5 * e_d2) + 5 * U32)
    else:
        r = torch.sqrt(d2)
        far = d2 > e_d2
        e_r = torch.where(far, e_d2 / (r + (d2 - e_d2).clamp_min(0.0).sqrt()).masked_fill(~far, 1.0), e_d2.sqrt()) + U32 * r
        if kernel_type == GP_MATERN12:
            k = torch.exp(-r)
            poly = torch.ones_like(d2)
            e_k = k * (torch.expm1(e_r) + 5 * U32)
        else:
            c = math.sqrt(3.0) if kernel_type == GP_MATERN32 else math.sqrt(5.0)
            cf = _f32(c)
            a = c * r
            e_a = abs(cf - c) * r + cf * e_r + U32 * cf * (r + e_r)
            ea = torch.exp(-a)
            if kernel_type == GP_MATERN32:
                poly = 1.0 + a
                k = poly * ea
                # (1 + a) e^-a: derivative a e^-a; 1 + a, os *, * expf round once each, expf 4 U32
                e_k = ea * torch.exp(e_a) * a * e_a + 7 * U32 * k
            else:
                b = 5.0 / 3.0 * d2
                poly = 1.0 + a + b
                k = poly * ea
                # (1 + a + b) e^-a moves with d2 through a and b at once: dk/dd2 = -e^-a (5/6 + 5 sqrt5 r / 6), finite at
                # r = 0.  The rounded constants and sqrtf move a (derivative (a + b) e^-a) and b (e^-a) on their own; the
                # polynomial rounds at most 2 U32 p
                e_a0 = abs(cf - c) * r + U32 * cf * 2.0 * r
                e_b0 = abs(_f32(5.0 / 3.0) - 5.0 / 3.0) * d2
                dk = 5.0 / 6.0 + 5.0 * c / 6.0 * (r + e_r)
                e_k = ea * torch.exp(e_a) * (dk * e_d2 + (a + b) * e_a0 + e_b0) + 8 * U32 * k
    K = osv * k
    E_K = osv * e_k + (2.0 * osv * poly + 0.5) * 2.0 ** -149
    eye = torch.eye(T, dtype=torch.bool, device=xd.device)
    nj = noise.double().view(B, 1, 1) + jit
    diag = osv + nj
    K = torch.where(eye, diag, K)
    E_K = torch.where(eye, U32 * (nj.abs() + diag.abs()), E_K)
    return K, E_K


def gp_factor(work, T):
    """The factor L [B, T, T] from the kernel's work buffer (work[b][c][r] = L[r][c], rows padded to ldw).  Entries above
    the diagonal outside the 32 x 32 diagonal blocks are never written: tril."""
    return torch.tril(work[:, :, :T].transpose(1, 2))


def gp_factor_residual(Lf, E_K):
    """L L^T in fp64 and its bound about the exact K + jitter I: |L L^T - K|_ij <= U32 d_ij (|L||L|^T)_ij + E_K,ij with
    d_ij = min(i, j) + 3.  For j = min(i, j), L_ij comes out of one sequential fp32 sum of K^_ij and j products: the c0
    products of the finished panels in the update's fmaf chain (c0 roundings), K^ - acc (one), the j - c0 products of
    the panel in the warp Cholesky or the row solve (one fmaf each); then L_ij = s * fl(1 / L_jj) (two roundings), s / L_jj
    (one) or sqrtf(s) (two on L_jj^2).  Pushing every rounding onto the products and L_ij L_jj (Higham, Lemma 8.4) leaves
    K^_ij exact and at most j + 3 relative errors on each term of sum_k<=j L_ik L_jk.  K^ itself is within E_K of K.
    A product or quotient that lands among the subnormals carries an absolute error of up to 2^-150 instead, once per
    rounding and scaled by L_jj where it is pushed onto L_ij L_jj: 2^-149 d_ij (1 + max(L_ii, L_jj))."""
    Ld = Lf.double()
    T = Ld.shape[-1]
    i = torch.arange(T, device=Ld.device)
    d = (torch.minimum(i.unsqueeze(1), i.unsqueeze(0)) + 3).double()
    La = Ld.abs()
    dg = torch.diagonal(La, dim1=-2, dim2=-1)
    floor = 2.0 ** -149 * d * (1.0 + torch.maximum(dg.unsqueeze(-1), dg.unsqueeze(-2)))
    return Ld @ Ld.transpose(-1, -2), U32 * d * (La @ La.transpose(-1, -2)) + E_K + floor


def gp_draw(Lf, z):
    """Exact y = L z from the kernel's own factor L [B, T, T] and z [B, T], and its bound
    U32 (32 + ceil((r + 1) / 32) + 1) sum_c |L_rc||z_c|: row r is one 32-term fmaf dot per panel it meets
    (ceil((r + 1) / 32) of them) added into y[r] in panel order."""
    Ld, zd = Lf.double(), z.double().unsqueeze(-1)
    T = Ld.shape[-1]
    r = torch.arange(T, device=Ld.device)
    d = (GP_PANEL + (r + GP_PANEL) // GP_PANEL + 1).double()
    return (Ld @ zd).squeeze(-1), U32 * d * (Ld.abs() @ zd.abs()).squeeze(-1)
