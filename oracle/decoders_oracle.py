"""fp64 restatement of the learned-temperature decoder heads (reference decoders.py:6-30) and per-element error bounds for
their row kernels (csrc/scaled_head.cu) -- TEST INFRASTRUCTURE ONLY.

`scaled_head` / `fixed_head` give every intermediate of a head's forward and backward in fp64.  The `*_bound` helpers follow
oracle/error_budget.py: the exact result in fp64 from the kernel's own inputs, and a bound c * bound on |got - exact| built
from the kernel's rounding steps and the depth of its sums (include/pfn_b200.h states the depths).  `head_bounds` composes
first-order magnitudes through the whole head, for comparing a head run end to end against the reference in fp64.
"""
import importlib.util
import math
import os

import torch

from oracle import error_budget as EB

HERE = os.path.dirname(os.path.abspath(__file__))
TEMPERATURES = (1., 1.4, 1.7, 2., 5., 10., 20., 40., 80., 160.)
TEMPS = torch.tensor(TEMPERATURES, dtype=torch.float32).double()    # the values the reference's float32 module uses
N_TEMPS = 10
# Constants c of the GPU tests, at least twice the worst ratio measured on an H100 80GB HBM3 (700 W power limit).  The row
# kernels' bounds are worst cases of their own rounding steps; a bf16 store alone reaches a ratio of 1.  The whole-head
# bounds are first-order magnitudes times HEAD_STEPS roundings of the storage unit, which random data reach a small
# fraction of.
C_HEAD = 2.0          # worst 0.996 (bf16 dz / dzz); fp32: dz 0.50, dzz 0.149, out 0.146, temp 0.128, dT 0.051, S 0.025
C_HEAD_WHOLE = 0.07   # worst 0.034 (FixedScaledDecoder fp32 mapper.2.bias); logits 0.0009, dhq 0.006
HEAD_STEPS = 8
GELU_GRAD_MAX = 1.13       # max |GELU'(x)|
GELU_CURV_MAX = 0.4        # max |GELU''(x)|


def load_reference():
    """The unmodified reference decoders.py vendored under oracle/_ref (oracle/build_ref.py), imported under a private
    name so that no top-level module is replaced; None when oracle/_ref has not been built."""
    path = os.path.join(HERE, "_ref", "decoders.py")
    if not os.path.isfile(path):
        return None
    spec = importlib.util.spec_from_file_location("_pfn_reference_decoders", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_grad(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


# ------------------------------------------------------------------------------------------------------------------
# fp64 restatement
# ------------------------------------------------------------------------------------------------------------------
def scaled_rows(zz, n_out, temps=TEMPS):
    """(out, temp, p) of ScaledDecoder's division from zz = [z | zt].  `temps`: the constants c (by default the fp32 values
    the reference's float32 module and the kernel use)."""
    zz = zz.double()
    z, zt = zz[:, :n_out], zz[:, n_out:n_out + N_TEMPS]
    p = torch.softmax(zt, -1)
    temp = p @ temps.double().to(zz.device)
    return z / temp.unsqueeze(-1), temp, p


def scaled_rows_bwd(g, zz, n_out, temps=TEMPS):
    """dzz = [g / temp | p (c - temp) dtemp] with dtemp = -(g . z) / temp^2."""
    g, zz = g.double(), zz.double()
    _, temp, p = scaled_rows(zz, n_out, temps)
    dtemp = -(g * zz[:, :n_out]).sum(-1) / temp ** 2
    dzt = p * (temps.double().to(zz.device) - temp.unsqueeze(-1)) * dtemp.unsqueeze(-1)
    return torch.cat([g / temp.unsqueeze(-1), dzt], -1)


def scaled_head(hq, W, b, W1, b1, W2, b2, gout=None, temps=TEMPS):
    """Every intermediate of ScaledDecoder's forward (and, given gout = dL/dlogits, backward) in fp64."""
    d = lambda t: t.double()
    hq, W, b, W1, b1, W2, b2 = map(d, (hq, W, b, W1, b1, W2, b2))
    n_out = W1.shape[0]
    r = {"u": hq @ W.T + b}
    r["g"] = gelu(r["u"])
    W12, b12 = torch.cat([W1, W2]), torch.cat([b1, b2])
    r["zz"] = r["g"] @ W12.T + b12
    r["out"], r["temp"], r["p"] = scaled_rows(r["zz"], n_out, temps)
    if gout is not None:
        r["dzz"] = scaled_rows_bwd(gout, r["zz"], n_out, temps)
        r["dW12"], r["db12"] = r["dzz"].T @ r["g"], r["dzz"].sum(0)
        r["du"] = (r["dzz"] @ W12) * gelu_grad(r["u"])
        r["dW"], r["db"], r["dhq"] = r["du"].T @ hq, r["du"].sum(0), r["du"] @ W
        r["grads"] = {"linear.weight": r["dW"], "linear.bias": r["db"], "linear1.weight": r["dW12"][:n_out],
                      "linear1.bias": r["db12"][:n_out], "linear2.weight": r["dW12"][n_out:], "linear2.bias": r["db12"][n_out:]}
    return r


def fixed_head(hq, W0, b0, W2, b2, T, gout=None):
    """Every intermediate of FixedScaledDecoder's forward (and backward) in fp64."""
    d = lambda t: t.double()
    hq, W0, b0, W2, b2, T = map(d, (hq, W0, b0, W2, b2, T))
    r = {"u": hq @ W0.T + b0}
    r["g"] = gelu(r["u"])
    r["zz"] = r["g"] @ W2.T + b2
    r["S"] = T.sum()
    r["out"] = r["zz"] / r["S"]
    if gout is not None:
        gout = gout.double()
        r["dzz"] = gout / r["S"]
        r["dT"] = torch.full_like(T, -(gout * r["zz"]).sum().item() / r["S"].item() ** 2)
        r["dW2"], r["db2"] = r["dzz"].T @ r["g"], r["dzz"].sum(0)
        r["du"] = (r["dzz"] @ W2) * gelu_grad(r["u"])
        r["dW0"], r["db0"], r["dhq"] = r["du"].T @ hq, r["du"].sum(0), r["du"] @ W0
        r["grads"] = {"mapper.0.weight": r["dW0"], "mapper.0.bias": r["db0"], "mapper.2.weight": r["dW2"],
                      "mapper.2.bias": r["db2"], "T": r["dT"]}
    return r


# ------------------------------------------------------------------------------------------------------------------
# row kernels: exact results from the kernel's own fp32 inputs and their bounds
# ------------------------------------------------------------------------------------------------------------------
def _temp_rel(zt):
    """Relative error bound of the kernel's temp: zt_k - max rounds (U32 |x_k|, hence U32 |x_k| relative in e_k), expf
    (2 ulp = 4 U32), the depth-5 butterfly sum of e (5 U32), the division e / s (U32), the products p c (U32) and the
    depth-5 sum of those (5 U32): p_k carries twice e's error, so U32 (2 max|x| + 20)."""
    x = zt - zt.max(-1, keepdim=True).values
    return EB.U32 * (2 * x.abs().max(-1).values + 20)


def scaled_fwd_bound(zz, n_out):
    """Exact (out, temp) from the kernel's input zz and their bounds."""
    zz = zz.double()
    out, temp, _ = scaled_rows(zz, n_out)
    rel = _temp_rel(zz[:, n_out:n_out + N_TEMPS])
    return {"out": out, "out_bound": (rel + EB.U32).unsqueeze(-1) * out.abs(), "temp": temp, "temp_bound": rel * temp}


def sum_depth(n_out):
    """Depth of a row's sum_j g_j z_j: fmaf over columns lane, lane + 32, ..., then the 5-level butterfly."""
    return (n_out + 31) // 32 + 5


def scaled_bwd_bound(g, zz, n_out, u_d):
    """Exact dzz [rows, n_out + 10] from the kernel's inputs g, zz, and its bound (u_d: unit roundoff of dzz's dtype).
    The kernel divides by its stored temp (relative error dT = _temp_rel), recomputes p (relative error dp), and forms
    dtemp from a sum of depth sum_depth(n_out), one squaring and one division."""
    g, zz = g.double(), zz.double()
    z, zt = zz[:, :n_out], zz[:, n_out:n_out + N_TEMPS]
    _, temp, p = scaled_rows(zz, n_out)
    exact = scaled_rows_bwd(g, zz, n_out)
    x = zt - zt.max(-1, keepdim=True).values
    rel_t = _temp_rel(zt).unsqueeze(-1)
    rel_p = EB.U32 * (2 * x.abs().max(-1).values + 14).unsqueeze(-1)
    t = temp.unsqueeze(-1)
    s_abs = (g * z).abs().sum(-1, keepdim=True)
    dtemp = -(g * z).sum(-1, keepdim=True) / t ** 2
    e_dtemp = EB.U32 * sum_depth(n_out) * s_abs / t ** 2 + dtemp.abs() * (2 * rel_t + 2 * EB.U32)
    cmt = (TEMPS.to(zz.device) - t).abs()
    dz_b = (rel_t + EB.U32 + u_d) * exact[:, :n_out].abs()
    dzt_b = p * (cmt * dtemp.abs() * (rel_p + 3 * EB.U32) + t * rel_t * dtemp.abs() + cmt * e_dtemp) \
        + u_d * exact[:, n_out:].abs()
    return exact, torch.cat([dz_b, dzt_b], -1)


def t_sum_depth(n_t):
    return (n_t + 255) // 256 + 8


def dot_depth(rows, n_out):
    """Depth of D = sum over rows of sum_j g_j z_j: the row sums, then thread-sequential over rows i, i + 1024, ...
    and a 10-level tree."""
    return sum_depth(n_out) + (rows + 1023) // 1024 + 10


def fixed_fwd_bound(z, T):
    """Exact (out, S) and their bounds; S's error is U32 depth sum|T|."""
    z, T = z.double(), T.double()
    S = T.sum()
    e_S = EB.U32 * t_sum_depth(T.numel()) * T.abs().sum()
    out = z / S
    return {"out": out, "out_bound": (e_S / S.abs() + EB.U32) * out.abs(), "S": S, "S_bound": e_S}


def fixed_bwd_bound(g, z, S, u_d):
    """Exact (dz, dT) from the kernel's inputs g, z and its S (fp32), and their bounds."""
    g, z, S = g.double(), z.double(), S.double().reshape(())
    dz = g / S
    D = (g * z).sum()
    dT = -D / S ** 2
    e_D = EB.U32 * dot_depth(g.shape[0], g.shape[1]) * (g * z).abs().sum()
    return {"dz": dz, "dz_bound": (EB.U32 + u_d) * dz.abs(), "dT": dT,
            "dT_bound": e_D / S ** 2 + 2 * EB.U32 * dT.abs()}


# ------------------------------------------------------------------------------------------------------------------
# whole heads: first-order magnitudes of every result, for a head run end to end against its fp64 restatement
# ------------------------------------------------------------------------------------------------------------------
def head_bounds(r, hq, W, b, W2nd, b2nd, u, scaled, n_out, gout):
    """{name: bound} for the logits, every parameter gradient and dhq of the head whose fp64 intermediates are r
    (scaled_head / fixed_head with gout).  Every stored operand and intermediate carries a relative error of at most u
    (the GEMM epilogues' fast GELU adds EB.GELU_ABS, the accumulations are far below); each is propagated through the
    head to first order with the magnitudes of the exact values, and the result is HEAD_STEPS u times that magnitude.
    W2nd, b2nd: the second layer's weight and bias (stacked [W1; W2] for ScaledDecoder)."""
    A = lambda t: t.double().abs()
    hq, W, b, W2nd, b2nd, gout = (t.double() for t in (hq, W, b, W2nd, b2nd, gout))
    u_mag = A(hq) @ A(W).T + A(b)
    g_mag = GELU_GRAD_MAX * u_mag + A(r["g"]) + EB.GELU_ABS / u
    zz_mag = g_mag @ A(W2nd).T + A(r["g"]) @ A(W2nd).T + A(b2nd)
    go = A(gout)
    if scaled:
        t, p = r["temp"].unsqueeze(-1), r["p"]
        cmt = (TEMPS.to(t.device) - t).abs()
        zt_mag = zz_mag[:, n_out:]
        t_mag = (p * cmt * zt_mag).sum(-1, keepdim=True) + t
        out_mag = zz_mag[:, :n_out] / t + A(r["zz"][:, :n_out]) * t_mag / t ** 2
        s = (gout * r["zz"][:, :n_out]).sum(-1, keepdim=True)
        s_mag = (go * zz_mag[:, :n_out]).sum(-1, keepdim=True)
        dtemp = s.abs() / t ** 2
        dtemp_mag = s_mag / t ** 2 + 2 * dtemp * t_mag / t
        p_mag = p * (zt_mag + (p * zt_mag).sum(-1, keepdim=True)) + p
        dzz_mag = torch.cat([go / t + go * t_mag / t ** 2,
                             p_mag * cmt * dtemp + p * (t_mag * dtemp + cmt * dtemp_mag)], -1)
    else:
        S = r["S"].abs()
        out_mag = zz_mag / S + A(r["zz"]) / S
        dzz_mag = 2 * go / S
    dzz = A(r["dzz"])
    dW2_mag = dzz_mag.T @ A(r["g"]) + dzz.T @ g_mag
    db2_mag = dzz_mag.sum(0)
    gp = gelu_grad(r["u"]).abs()
    dg = dzz @ A(W2nd)
    du_mag = (dzz_mag @ A(W2nd) + dg) * gp + dg * (GELU_CURV_MAX * u_mag + EB.GELU_GRAD_ABS / u)
    du = A(r["du"])
    k = HEAD_STEPS * u
    out = {"out": k * out_mag, "dW2": k * dW2_mag, "db2": k * db2_mag, "dW": k * (du_mag.T @ A(hq) + du.T @ A(hq)),
           "db": k * du_mag.sum(0), "dhq": k * (du_mag @ A(W) + du @ A(W))}
    if not scaled:
        # dT = -sum(g z) / S^2: z's error through the dot product, S's through the square
        out["dT"] = k * ((go * zz_mag).sum() + 2 * (gout * r["zz"]).sum().abs()) / S ** 2
    return out
