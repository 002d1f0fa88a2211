"""fp64 restatement of encoders.Conv and per-element bounds of its kernels -- TEST INFRASTRUCTURE ONLY.

The module in fp64 (`forward`, `gradients`) is stated with torch.nn.functional.conv2d / relu / mean / linear in NCHW.  The
bounds take each kernel's own (already rounded) NHWC inputs and state its 3x3 convolution as the GEMM over the im2col
view (columns ordered (tap, ci), tap = 3 dr + dc, K = 9 C_in), so that error_budget.gemm gives the exact result and the
bound |got - exact| <= c (u |exact| + c_acc U32 K |A||B|) element by element (error_budget's module docstring).
"""
import torch
import torch.nn.functional as Fn

from . import error_budget as eb

# Constants c of the GPU tests (tests/test_gpu_conv_encoder.py), at least twice the worst ratio measured on an H100 80GB
# HBM3 (DESIGN.md section 3.1 lists the ratios)
C_CONV = 2.0          # conv forward and data gradient results (worst 0.996, bf16 output; fp32 0.40, input conv)
C_ACC_CONV = 0.1      # wgmma kernels: fp32 accumulation over K = 9 C_in (+ the bias) in units of U32 K |A||B| (their
                      # bf16 results are bound by the output rounding; the fp32 64 -> 64 paths reach 0.011 of C_CONV)
# The direct FMA kernels (the input conv, the fp32 path) sum K = 9 C_in + 1 terms in sequence: the worst case of such a
# sum is 1 in these units, and the ten-term input conv comes near it (ratio 2.2 against C_ACC_CONV)
C_ACC_CONV_DIRECT = 1.0
C_ACC_CONV_WGRAD = 0.3  # weight and bias gradients: fp32 sums over every output pixel (worst 0.27 of this, i.e. 0.08)
C_MEAN = 2.0          # spatial mean and its backward (worst 0.996, bf16 mean; backward 0.87)


def n_conv(S):
    return min(5, (S - 2) // 2)


def _pairs(params):
    return [params[i:i + 2] for i in range(0, len(params) - 2, 2)], params[-2:]


def forward(x, params, S):
    """x [N, S*S]; params (w, b) per applied conv then (linear weight, bias).  Returns (out [N, E], post-ReLU activations
    NCHW, feat [N, 64]), all fp64."""
    convs, (lw, lb) = _pairs([p.double() for p in params])
    h = x.double().reshape(-1, 1, S, S)
    acts = []
    for w, b in convs:
        h = torch.relu(Fn.conv2d(h, w, b))
        acts.append(h)
    feat = h.mean((2, 3))
    return Fn.linear(feat, lw, lb), acts, feat


def gradients(x, params, S, dout):
    """(out, [d param for param in params]) of sum(out * dout) in fp64."""
    leaves = [p.detach().double().requires_grad_(True) for p in params]
    out, _, _ = forward(x, leaves, S)
    grads = torch.autograd.grad(out, leaves, dout.double())
    return out.detach(), list(grads)


def im2col(x):
    """x [N, s, s, C] -> [N (s-2)^2, 9 C], column tap * C + ci holding x[n, r + dr, c + dc, ci]."""
    s = x.shape[1]
    cols = [x[:, dr:dr + s - 2, dc:dc + s - 2, :] for dr in range(3) for dc in range(3)]
    return torch.stack(cols, 3).reshape(-1, 9 * x.shape[-1])


def _with_ones(A, B, b):
    """[A, 1] and [B, b]: the bias as one more term of the contraction (the direct kernels start their sums from it)."""
    one = torch.ones(A.shape[0], 1, dtype=A.dtype, device=A.device)
    return torch.cat([A, one], 1), torch.cat([B, b.reshape(-1, 1).to(B.dtype)], 1)


def conv_fwd(x, W, b, u_out, c_acc=C_ACC_CONV):
    """relu(conv(x, W) + b) of one kernel launch: x [N, s, s, C] (its own input), W [64, C, 3, 3], b [64].
    Returns (exact, bound) as [N, s-2, s-2, 64]."""
    N, s = x.shape[0], x.shape[1]
    A, B = _with_ones(im2col(x), W.permute(0, 2, 3, 1).reshape(W.shape[0], -1), b)
    val, bound, _ = eb.gemm(A, B, u_out, c_acc)
    shape = (N, s - 2, s - 2, W.shape[0])
    return torch.relu(val).reshape(shape), bound.reshape(shape)


def conv_dgrad(gpad, W, x, u_out, c_acc=C_ACC_CONV):
    """(input gradient of the 64 -> 64 layer) * [x > 0]: gpad [N, s+2, s+2, 64] the padded output gradient the kernel
    read, x [N, s, s, 64] the layer's input.  Returns (exact, bound) as [N, s, s, 64] (the padded output's interior)."""
    N, s = x.shape[0], x.shape[1]
    B = W.flip(2, 3).permute(1, 2, 3, 0).reshape(W.shape[1], -1)
    mask = (x.reshape(-1, x.shape[-1]) > 0).to(torch.float64)
    val, bound, _ = eb.gemm(im2col(gpad), B, u_out, c_acc, aux=mask, epilogue="mul")
    return val.reshape(x.shape), bound.reshape(x.shape)


def conv_wgrad(g, x, c_acc=C_ACC_CONV_WGRAD, block_k=1 << 16):
    """(dW [64, C, 3, 3], db [64]) exact and bound (fp32 results): g [N, s-2, s-2, 64] the output gradient (unpadded),
    x [N, s, s, C] the layer's input."""
    C = x.shape[-1]
    gm = g.reshape(-1, g.shape[-1]).float()            # bf16 and fp32 values are exact in fp32
    A = gm.t()
    Bt = torch.cat([im2col(x.float()), torch.ones(gm.shape[0], 1, device=gm.device)], 1)
    val, bound, _ = eb.gemm(A, Bt.t(), eb.U32, c_acc, block_k=block_k)

    def split(t):
        return t[:, :-1].reshape(-1, 3, 3, C).permute(0, 3, 1, 2), t[:, -1]
    (dw, db), (bw, bb) = split(val), split(bound)
    return dw, db, bw, bb


def mean_fwd(y, u_out):
    """feat [N, 64] = mean of y [N, s, s, 64] over its pixels: four strided partial sums of P / 4 terms, three adds, a
    division."""
    P = y.shape[1] * y.shape[2]
    yd = y.double().reshape(y.shape[0], P, -1)
    exact = yd.mean(1)
    return exact, u_out * exact.abs() + eb.U32 * (P / 4 + 4) * yd.abs().mean(1)


def mean_bwd(dfeat, y, u_out):
    """g [N, s, s, 64] = dfeat / s^2 * [y > 0] (the interior of the padded gradient)."""
    P = y.shape[1] * y.shape[2]
    exact = (dfeat.double() / P)[:, None, None, :] * (y > 0).double()
    return exact, (u_out + eb.U32) * exact.abs()
