"""The PFN step engine: explicit forward/backward of the post-norm GELU encoder stack, the embedding stage and
the decoder head, expressed as sequences of C-ABI kernel calls (libpfn_b200.so) and exposed to PyTorch as three
`torch.autograd.Function`s so that `loss.backward()` in the reference-shaped `train.train` keeps working.

Restates what the reference obtains from `nn.TransformerEncoder` (reference transformer.py:17-18,84;
torch nn/modules/transformer.py:951-982).

Layout: activations are [T*B, cols] row-major with token row = t*B + b (the reference's sequence-first layout,
flattened), in the activation dtype (bf16 by default, fp32 in parity mode).  Parameters stay fp32 masters; the
bf16 mode casts them once per forward.  Weight gradients are produced in fp32 by split-K tensor-core GEMMs that
read dY and X *in place* as MN-major operands (no transposed copies).
"""
import os

import torch

from . import _lib as L

LAYER_PARAM_NAMES = ("in_w", "in_b", "out_w", "out_b", "w1", "b1", "w2", "b2", "g1", "be1", "g2", "be2")
N_LAYER_PARAMS = len(LAYER_PARAM_NAMES)
LN_EPS = 1e-5


# Data-parallel hook (parallel.OverlappedGradReducer): when set, it is called from inside the backward passes as soon as a
# bucket of parameter gradients is complete in stream order -- `hook(flat_fp32_bucket)` -- so that its all-reduce overlaps the
# rest of the backward; `GRAD_BUCKET_SYNC()` is called before the gradients are handed to autograd.
_DELTA_FUSION = os.environ.get("PFN_B200_DELTA_FUSION", "1") != "0"     # A/B knob (tools/ab_env.sh)
GRAD_BUCKET_HOOK = None
GRAD_BUCKET_SYNC = None


def default_precision():
    return os.environ.get("PFN_B200_PRECISION", "bf16")


def act_dtype(precision):
    if precision == "bf16":
        return torch.bfloat16
    if precision == "fp32":
        return torch.float32
    raise ValueError(f"precision must be 'bf16' or 'fp32', got {precision!r}")


def _wgrad_splits(n_tokens, out_rows, out_cols):
    """Split-K factor of a wgrad GEMM (contraction over the tokens): about two work units (128 x 128 tile, k-split) per
    SM.  The persistent GEMM runs one CTA per SM whose two consumer warpgroups take the CTA's units in turn, so two units
    per CTA keep the tensor pipe busy from the first main loop to the last while the first unit's fp32 reduce-add
    epilogue overlaps the second's main loop; more splits only add reduce-add traffic on the same
    [out_rows, out_cols] block (tools/sweep_wgrad_splits.py times the alternatives)."""
    tiles = ((out_rows + 127) // 128) * ((out_cols + 127) // 128)
    units = 2 * L.num_sms()
    num_kb = (n_tokens + 63) // 64
    want = max(1, units // max(tiles, 1))
    return max(1, min(want, num_kb // 8 if num_kb >= 16 else 1))


def site_seed(seed, layer, site):
    """Seed of one dropout site (0 attention probabilities, 1 attention block output, 2 after GELU, 3 MLP block output)
    of one layer, derived from the step's seed."""
    return (int(seed) + 0x9E3779B9 * (4 * layer + site + 1)) & 0xFFFFFFFF


def _cast(w, dtype):
    """Operand copy of a weight in the activation dtype: the optimizer's bf16 shadow (optim.FusedClipAdam rewrites it inside
    the update kernel) when it mirrors the current version of the parameter, else a cast."""
    from .optim import cast_weight
    return cast_weight(w, dtype)


def _linear_fwd(x, w_c, bias, *, aux=None, epilogue=L.EPI_NONE, want_pre=False, out_dtype=None):
    """y = epi(x @ w_c^T + bias) (+aux).  x [M,K], w_c [N,K] (activation dtype)."""
    M, N = x.shape[0], w_c.shape[0]
    y = torch.empty(M, N, device=x.device, dtype=out_dtype or x.dtype)
    pre = torch.empty(M, N, device=x.device, dtype=x.dtype) if want_pre else None
    L.gemm(x, w_c, y, bias=bias, aux=aux, C2=pre, epilogue=epilogue)
    return (y, pre) if want_pre else y


_GELU_GRAD_FWD = os.environ.get("PFN_B200_GELU_GRAD_FWD", "1") != "0"     # A/B knob (tools/ab_env.sh)


def _gelu_linear_fwd(x, w_c, bias):
    """(gelu(x @ w_c^T + bias), s, s_is_grad): what the backward needs of the GELU is either the pre-activation u
    (s_is_grad False: the dgrad epilogue evaluates gelu'(u)) or, on the tensor-core path, gelu'(u) itself, produced by the
    forward epilogue from the sigmoid it has already computed -- the backward dgrad then only multiplies (the epilogues are
    bound by instruction issue, and gelu' alone is ~14 instructions per element)."""
    M, N = x.shape[0], w_c.shape[0]
    y = torch.empty(M, N, device=x.device, dtype=x.dtype)
    s = torch.empty(M, N, device=x.device, dtype=x.dtype)
    as_grad = _GELU_GRAD_FWD and L.tc_gemm_ok(x, w_c, y, None, s)
    L.gemm(x, w_c, y, bias=bias, C2=s, epilogue=L.EPI_GELU, c2_gelu_grad=as_grad)
    return y, s, as_grad


def _gelu_linear_dgrad(dy, w_c, s, s_is_grad):
    """dx = (dy @ w_c) * gelu'(u), with s = gelu'(u) (s_is_grad) or s = u."""
    return _linear_dgrad(dy, w_c, aux=s, epilogue=L.EPI_MUL if s_is_grad else L.EPI_GELU_BWD)


def _linear_dgrad(dy, w_c, *, aux=None, epilogue=L.EPI_NONE, rowdot=None):
    """dx = dy @ w_c (+aux | * gelu'(aux) | with rowdot[0][m, k // rowdot[1]] += sum_k dx[m,k] aux[m,k]).
    dy [M,N], w_c [N,K] read as an MN-major B operand."""
    M, K = dy.shape[0], w_c.shape[1]
    dx = torch.empty(M, K, device=dy.device, dtype=dy.dtype)
    L.gemm(dy, w_c, dx, b_mn_major=True, aux=aux, epilogue=epilogue, M=M, N=K, K=w_c.shape[0], rowdot=rowdot)
    return dx


def _linear_wgrad(dy, x, dw, rows=None, cols=None):
    """dw[N,K] += dy^T @ x.  dy [M,N], x [M,K] both read in place as MN-major operands; fp32 split-K (TMA reduce-add)."""
    n_tok = dy.shape[0]
    N = dw.shape[0] if rows is None else rows
    K = dw.shape[1] if cols is None else cols
    L.gemm(dy, x, dw, a_mn_major=True, b_mn_major=True, accumulate=True, k_splits=_wgrad_splits(n_tok, N, K),
           M=N, N=K, K=n_tok)


class EncoderStackFn(torch.autograd.Function):
    """src [T*B, E] (activation dtype) -> output of `nlayers` post-norm encoder layers under the sep mask."""

    @staticmethod
    def forward(ctx, src, T, B, sep, nhead, precision, keep, drop, *params):
        """`keep`: the CALLER's grad mode (torch.is_grad_enabled() outside this Function — inside it is always off, and
        ctx.needs_input_grad does not reflect no_grad); when False no activation is retained (inference memory).
        `drop`: None or (seed, thr) — training-mode dropout with probability thr/256 at the reference layer's four sites
        (attention probabilities, attention block output, after the GELU, MLP block output; torch
        nn/modules/transformer.py:961-982).  Masks are counter-based and regenerated in backward (csrc/dropout.cuh)."""
        L.require_cuda(src, *params)
        dt = act_dtype(precision)
        assert src.dtype == dt and src.dim() == 2
        n_layers = len(params) // N_LAYER_PARAMS
        N, E = src.shape
        dh = E // nhead
        keep = bool(keep) and any(ctx.needs_input_grad)
        saved = []
        h = src.contiguous()
        thr = drop[1] if drop else 0
        for li in range(n_layers):
            P = dict(zip(LAYER_PARAM_NAMES, params[li * N_LAYER_PARAMS:(li + 1) * N_LAYER_PARAMS]))
            in_w, out_w, w1, w2 = (_cast(P[k], dt) for k in ("in_w", "out_w", "w1", "w2"))
            qkv = _linear_fwd(h, in_w, P["in_b"])
            attn = torch.empty(N, E, device=h.device, dtype=dt)
            lse = torch.empty(B * nhead, T, device=h.device, dtype=torch.float32)
            L.attention_fwd(qkv, attn, lse, T, B, nhead, dh, sep, drop=(site_seed(drop[0], li, 0), thr) if thr else None)
            if thr:
                z1 = _linear_fwd(attn, out_w, P["out_b"])
                L.dropout(z1, z1, site_seed(drop[0], li, 1), thr, residual=h)           # h + dropout1(attn block)
            else:
                z1 = _linear_fwd(attn, out_w, P["out_b"], aux=h)
            h1 = torch.empty_like(z1)
            mean1 = torch.empty(N, device=h.device, dtype=torch.float32)
            rstd1 = torch.empty_like(mean1)
            L.layernorm_fwd(z1, P["g1"], P["be1"], h1, mean1, rstd1, LN_EPS)
            g, u, u_is_grad = _gelu_linear_fwd(h1, w1, P["b1"])
            if thr:
                L.dropout(g, g, site_seed(drop[0], li, 2), thr)                           # dropout(GELU(.)), in place
                z2 = _linear_fwd(g, w2, P["b2"])
                L.dropout(z2, z2, site_seed(drop[0], li, 3), thr, residual=h1)          # h1 + dropout2(MLP block)
            else:
                z2 = _linear_fwd(g, w2, P["b2"], aux=h1)
            h2 = torch.empty_like(z2)
            mean2 = torch.empty_like(mean1)
            rstd2 = torch.empty_like(mean1)
            L.layernorm_fwd(z2, P["g2"], P["be2"], h2, mean2, rstd2, LN_EPS)
            if keep:
                # the activation-dtype weight copies are kept for the backward as well (4 small tensors per layer) instead of
                # being cast a second time there
                saved.append((h, qkv, attn, lse, z1, mean1, rstd1, h1, u, g, z2, mean2, rstd2, in_w, out_w, w1, w2))
            h = h2
        ctx.saved_acts = saved
        ctx.u_is_grad = u_is_grad if n_layers else False        # same decision for every layer (same shapes / dtypes)
        ctx.params = params
        ctx.meta = (T, B, sep, nhead, precision, n_layers)
        ctx.drop = drop if thr else None
        return h

    @staticmethod
    def backward(ctx, dout):
        if ctx.saved_acts is None:
            raise RuntimeError("EncoderStackFn: activations were already released by a previous backward "
                               "(the engine frees them layer by layer; retain_graph=True is not supported)")
        T, B, sep, nhead, precision, n_layers = ctx.meta
        dt = act_dtype(precision)
        params = ctx.params
        dev = dout.device
        N, E = dout.shape
        dh = E // nhead
        sizes = [p.numel() for p in params]
        flat = torch.zeros(sum(sizes), device=dev, dtype=torch.float32)
        grads, off = [], 0
        for p, n in zip(params, sizes):
            grads.append(flat[off:off + n].view(p.shape))
            off += n
        dh2 = dout.contiguous().to(dt)
        for li in reversed(range(n_layers)):
            P = dict(zip(LAYER_PARAM_NAMES, params[li * N_LAYER_PARAMS:(li + 1) * N_LAYER_PARAMS]))
            G = dict(zip(LAYER_PARAM_NAMES, grads[li * N_LAYER_PARAMS:(li + 1) * N_LAYER_PARAMS]))
            h, qkv, attn, lse, z1, mean1, rstd1, h1, u, g, z2, mean2, rstd2, in_w, out_w, w1, w2 = ctx.saved_acts[li]
            ctx.saved_acts[li] = None
            # ---- LN2 and the MLP
            drop = ctx.drop
            dz2 = torch.empty_like(z2)
            L.layernorm_bwd(dh2, z2, mean2, rstd2, P["g2"], dz2, G["g2"], G["be2"], None if drop else G["b2"])
            del dh2, z2
            dm = dz2
            if drop:        # the MLP block saw dropout2: its output gradient is the masked, rescaled dz2 (residual keeps dz2)
                dm = torch.empty_like(dz2)
                L.dropout(dz2, dm, site_seed(drop[0], li, 3), drop[1])
                L.colsum(dm, G["b2"])
            _linear_wgrad(dm, g, G["w2"])
            du = _gelu_linear_dgrad(dm, w2, u, ctx.u_is_grad)
            if drop:
                L.dropout(du, du, site_seed(drop[0], li, 2), drop[1])       # mask of dropout(GELU(u)) commutes with GELU'(u)
            del g, u, dm
            L.colsum(du, G["b1"])
            _linear_wgrad(du, h1, G["w1"])
            dh1 = _linear_dgrad(du, w1, aux=dz2)
            del du, dz2, h1
            # ---- LN1 and attention
            dz1 = torch.empty_like(z1)
            L.layernorm_bwd(dh1, z1, mean1, rstd1, P["g1"], dz1, G["g1"], G["be1"], None if drop else G["out_b"])
            del dh1, z1
            da = dz1
            if drop:
                da = torch.empty_like(dz1)
                L.dropout(dz1, da, site_seed(drop[0], li, 1), drop[1])
                L.colsum(da, G["out_b"])
            _linear_wgrad(da, attn, G["out_w"])
            tc_attn = L.tc_attention_ok(qkv, dh)
            fuse_delta = tc_attn and _DELTA_FUSION and L.tc_gemm_ok(da, out_w, attn, attn)
            if fuse_delta:
                # delta = rowsum(dO * O) per (token, head) falls out of the out-projection dgrad's epilogue (the thread that
                # holds a row of dO for one head multiplies it with the O row it reads as `aux`): no separate pass over O and dO
                delta = torch.zeros(N, nhead, device=dev, dtype=torch.float32)
                dattn = _linear_dgrad(da, out_w, aux=attn, epilogue=L.EPI_ROWDOT, rowdot=(delta, dh))
            else:
                delta = torch.empty_like(lse)
                dattn = _linear_dgrad(da, out_w)
            del da
            dqkv = torch.empty_like(qkv)
            fused_bias = (not drop) and tc_attn
            L.attention_bwd(qkv, attn, lse, dattn, dqkv, delta, T, B, nhead, dh, sep,
                            drop=(site_seed(drop[0], li, 0), drop[1]) if drop else None,
                            dq_colsum=G["in_b"][:E] if fused_bias else None, delta_token_major=fuse_delta)
            del dattn, attn, qkv
            if fused_bias:
                # in-projection bias gradient without re-reading dqkv (1.5 GB per layer at cfg 2): the q third comes out of
                # the dQ kernel's staged tiles; the k third is zero in exact arithmetic (each row of dS sums to zero, so
                # sum_j dK_j = sum_i (sum_j dS_ij) q_i = 0 -- the reference's value is rounding noise); the v third is
                # sum_j dV_j = sum_i (sum_j P_ij) dO_i = colsum(dO) = colsum(dz1) W_out, and colsum(dz1) is the out_proj
                # bias gradient the LayerNorm backward just produced.
                G["in_b"][2 * E:] += G["out_b"] @ P["out_w"].detach().float()
            else:
                L.colsum(dqkv, G["in_b"])
            _linear_wgrad(dqkv, h, G["in_w"])
            dh2 = _linear_dgrad(dqkv, in_w, aux=dz1)
            del dqkv, dz1, h
            if GRAD_BUCKET_HOOK is not None:       # this layer's 12 gradients are one contiguous slice of the flat buffer
                lo = sum(sizes[:li * N_LAYER_PARAMS])
                GRAD_BUCKET_HOOK(flat[lo:lo + sum(sizes[li * N_LAYER_PARAMS:(li + 1) * N_LAYER_PARAMS])])
        if GRAD_BUCKET_SYNC is not None:
            GRAD_BUCKET_SYNC()
        ctx.saved_acts = None
        return (dh2, None, None, None, None, None, None, None) + tuple(grads)


class EmbedFn(torch.autograd.Function):
    """(x [T,B,F], y [T,B]) -> src [T*B, E]:  x Wx^T + bx + (t < sep)(y wy + by)   (reference transformer.py:68-74)."""

    @staticmethod
    def forward(ctx, x, y, Wx, bx, wy, by, sep, precision):
        L.require_cuda(x, y, Wx, bx, wy, by)
        T, B, F = x.shape
        E = Wx.shape[0]
        x = x.detach().contiguous().float()
        y = y.detach().contiguous().float()
        out = torch.empty(T * B, E, device=x.device, dtype=act_dtype(precision))
        L.embed_fwd(x, y, Wx.detach().contiguous(), bx.detach().contiguous(), wy.detach().contiguous().view(-1),
                    by.detach().contiguous(), out, T, B, F, E, sep)
        ctx.save_for_backward(x, y)
        ctx.meta = (T, B, F, E, sep, wy.shape)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, y = ctx.saved_tensors
        T, B, F, E, sep, wy_shape = ctx.meta
        dev = dout.device
        dWx = torch.zeros(E, F, device=dev)
        dbx = torch.zeros(E, device=dev)
        dwy = torch.zeros(E, device=dev)
        dby = torch.zeros(E, device=dev)
        L.embed_bwd(dout.contiguous(), x, y, dWx, dbx, dwy, dby, T, B, F, E, sep)
        return None, None, dWx, dbx, dwy.view(wy_shape), dby, None, None


class DecoderFn(torch.autograd.Function):
    """hq [Nq, E] -> logits [Nq, n_out] fp32:  GELU(hq W0^T + b0) W2^T + b2  (reference transformer.py:23,85),
    applied to the query rows only (the reference computes all T rows and slices, transformer.py:91)."""

    @staticmethod
    def forward(ctx, hq, W0, b0, W2, b2, precision):
        L.require_cuda(hq, W0, b0, W2, b2)
        dt = act_dtype(precision)
        hq = hq.contiguous()
        w0, w2 = _cast(W0, dt), _cast(W2, dt)
        n_out = W2.shape[0]
        g, u, u_is_grad = _gelu_linear_fwd(hq, w0, b0)
        ld = (n_out + 3) // 4 * 4
        logits_buf = torch.empty(hq.shape[0], ld, device=hq.device, dtype=torch.float32)
        logits = logits_buf[:, :n_out]
        L.gemm(g, w2, logits, bias=b2.detach().contiguous())
        ctx.save_for_backward(hq, u, g, W0, W2, w0, w2)
        ctx.u_is_grad = u_is_grad
        ctx.precision = precision
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        hq, u, g, W0, W2, w0, w2 = ctx.saved_tensors
        dt = act_dtype(ctx.precision)
        dev = dlogits.device
        Nq, n_out = dlogits.shape
        ld = (n_out + 7) // 8 * 8
        dl = torch.zeros(Nq, ld, device=dev, dtype=dt)
        dl[:, :n_out] = dlogits
        dlv = dl[:, :n_out]
        sizes = [W0.numel(), W0.shape[0], W2.numel(), n_out]
        flat = torch.zeros(sum(sizes), device=dev, dtype=torch.float32)        # one bucket: a single all-reduce under DP
        dW0 = flat[:sizes[0]].view(W0.shape)
        db0 = flat[sizes[0]:sizes[0] + sizes[1]]
        dW2 = flat[sizes[0] + sizes[1]:sizes[0] + sizes[1] + sizes[2]].view(W2.shape)
        db2 = flat[sizes[0] + sizes[1] + sizes[2]:]
        L.colsum(dlv, db2)
        _linear_wgrad(dlv, g, dW2)
        du = _gelu_linear_dgrad(dlv, w2, u, ctx.u_is_grad)
        L.colsum(du, db0)
        _linear_wgrad(du, hq, dW0)
        dhq = _linear_dgrad(du, w0)
        if GRAD_BUCKET_HOOK is not None:
            GRAD_BUCKET_HOOK(flat)
            GRAD_BUCKET_SYNC()     # 2 MB bucket: wait for it (stream-level) so autograd never touches a buffer NCCL is still writing
        return dhq, dW0, db0, dW2, db2, None


def layer_params(layer):
    """The 12 parameter tensors of one nn.TransformerEncoderLayer in LAYER_PARAM_NAMES order."""
    return (layer.self_attn.in_proj_weight, layer.self_attn.in_proj_bias, layer.self_attn.out_proj.weight,
            layer.self_attn.out_proj.bias, layer.linear1.weight, layer.linear1.bias, layer.linear2.weight,
            layer.linear2.bias, layer.norm1.weight, layer.norm1.bias, layer.norm2.weight, layer.norm2.bias)
