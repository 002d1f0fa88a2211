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
C_ACC_SIMT = 0.35


def check(name, got, exact, bound, c):
    """Assert |got - exact| <= c * bound elementwise; print and return the worst ratio.  Where the bound is 0 the
    kernel must be exact."""
    err = (got.double() - exact.double()).abs()
    bound = bound.double().expand_as(err)
    if (err[bound == 0] > 0).any():
        raise AssertionError(f"{name}: nonzero error where the bound is 0")
    ratio = (err / bound.clamp_min(1e-300)).masked_fill(bound == 0, 0.0)
    worst = ratio.max().item() if ratio.numel() else 0.0
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


def attention_bwd(f, dout, out_kernel):
    """Exact dQ, dK, dV (token-major [T*B, E] each) of the forward `f` for the upstream gradient dout, and their bounds.

    dS = P (dP - delta) with dP = keep drop_scale dO V^T and delta_i = dO_i . out_i.  The kernel rounds P and dS to the
    storage type before the second MMAs and the results at the end, so with |dS|~ = P (|dP| + |delta|):
      dV: unit P^^T |dO|
      dQ: scale (unit |dS|~ |K| + e_delta P |K|)
      dK: scale (|dS|~^T (unit |Q|) + P^T (e_delta |Q|))
    where e_delta,i = |dO_i . (out_kernel - out_exact)_i| is the error the kernel inherits by forming delta from the
    output it stored (not a rounding of its own, so it is not scaled by u)."""
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
    e_delta = (do * (_heads(out_kernel.double(), T, B, H, dh) - out)).sum(-1, keepdim=True).abs()
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
