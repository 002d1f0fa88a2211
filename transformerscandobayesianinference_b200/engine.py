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

from . import _lib as L, _lib_input_grad as LIG, _lib_ragged as LR, _lib_ragged_train as LRT

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


def _flat_grads(dev, *shapes):
    """One zeroed fp32 buffer holding gradients of the given shapes back to back (a single all-reduce under DP), and
    views of it in that order."""
    sizes = [torch.Size(s).numel() for s in shapes]
    flat = torch.zeros(sum(sizes), device=dev, dtype=torch.float32)
    views, off = [], 0
    for s, n in zip(shapes, sizes):
        views.append(flat[off:off + n].view(s))
        off += n
    return flat, views


def _bucket_ready(flat, wait=True):
    """Hand a complete bucket of gradients to the data-parallel hook, if one is set.  `wait`: then wait for it
    (stream-level) so autograd never touches a buffer NCCL is still writing; the encoder stack waits once, after its
    last layer's bucket."""
    if GRAD_BUCKET_HOOK is not None:
        GRAD_BUCKET_HOOK(flat)
        if wait:
            GRAD_BUCKET_SYNC()


class RaggedSeps:
    """One single_eval_pos per dataset, in place of the scalar `sep` of EncoderStackFn and EmbedFn: `n_keys` the int32 [B]
    device tensor of the values, `s_min` / `s_max` their least and greatest value (host ints)."""
    __slots__ = ("n_keys", "s_min", "s_max")

    def __init__(self, n_keys, s_min, s_max):
        self.n_keys, self.s_min, self.s_max = n_keys, int(s_min), int(s_max)


def _attention_fwd(qkv, attn, lse, T, B, nhead, dh, sep, drop):
    """The masked attention forward at the scalar sep, or at one separator per dataset (RaggedSeps)."""
    if isinstance(sep, RaggedSeps):
        LRT.attention_ragged_train_fwd(qkv, attn, lse, T, B, nhead, dh, sep.s_max, sep.n_keys, drop=drop)
    else:
        L.attention_fwd(qkv, attn, lse, T, B, nhead, dh, sep, drop=drop)


def _attention_bwd(qkv, attn, lse, dattn, dqkv, delta, T, B, nhead, dh, sep, **kw):
    """The backward of _attention_fwd."""
    if isinstance(sep, RaggedSeps):
        LRT.attention_ragged_train_bwd(qkv, attn, lse, dattn, dqkv, delta, T, B, nhead, dh, sep.s_max, sep.n_keys, **kw)
    else:
        L.attention_bwd(qkv, attn, lse, dattn, dqkv, delta, T, B, nhead, dh, sep, **kw)


def _stack_start(src, precision, nhead, params, kv=None):
    """Checks of an encoder stack call; (activation dtype, number of layers, head dim, contiguous src)."""
    L.require_cuda(src, kv, *params)
    dt = act_dtype(precision)
    assert src.dtype == dt and src.dim() == 2 and (kv is None or kv.dtype == dt)
    return dt, len(params) // N_LAYER_PARAMS, src.shape[1] // nhead, src.contiguous()


def _layer(seq, li):
    """Layer li's entries of a sequence with one entry per stack parameter (the parameters, their gradients), by name."""
    return dict(zip(LAYER_PARAM_NAMES, seq[li * N_LAYER_PARAMS:(li + 1) * N_LAYER_PARAMS]))


def _layer_qkv(h, params, li, dt):
    """Layer li's parameters by name, its four weight matrices in the activation dtype, its in-projection
    qkv = h W_in^T + b_in, and an uninitialised attention output buffer."""
    P = _layer(params, li)
    in_w, out_w, w1, w2 = (_cast(P[k], dt) for k in ("in_w", "out_w", "w1", "w2"))
    qkv = _linear_fwd(h, in_w, P["in_b"])
    return P, (in_w, out_w, w1, w2), qkv, torch.empty_like(h)


def _layer_tail(h, attn, P, out_w, w1, w2, drop, li):
    """One encoder layer after its attention: z1 = h + attn W_out^T + b_out, h1 = LN1(z1), g = GELU(h1 W1^T + b1),
    z2 = h1 + g W2^T + b2, h2 = LN2(z2), with dropout at the last three sites when `drop` is set.  Returns
    (z1, mean1, rstd1, h1, u, u_is_grad, g, z2, mean2, rstd2, h2)."""
    N = h.shape[0]
    thr = drop[1] if drop else 0
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
    return z1, mean1, rstd1, h1, u, u_is_grad, g, z2, mean2, rstd2, h2


class EncoderStackFn(torch.autograd.Function):
    """src [T*B, E] (activation dtype) -> output of `nlayers` post-norm encoder layers under the sep mask; `sep` is an int
    or a RaggedSeps (dataset b's rows then attend under its own separator).  Only the attention depends on sep."""

    @staticmethod
    def forward(ctx, src, T, B, sep, nhead, precision, keep, drop, *params):
        """`keep`: the CALLER's grad mode (torch.is_grad_enabled() outside this Function — inside it is always off, and
        ctx.needs_input_grad does not reflect no_grad); when False no activation is retained (inference memory).
        `drop`: None or (seed, thr) — training-mode dropout with probability thr/256 at the reference layer's four sites
        (attention probabilities, attention block output, after the GELU, MLP block output; torch
        nn/modules/transformer.py:961-982).  Masks are counter-based and regenerated in backward (csrc/dropout.cuh)."""
        dt, n_layers, dh, h = _stack_start(src, precision, nhead, params)
        keep = bool(keep) and any(ctx.needs_input_grad)
        saved = []
        thr = drop[1] if drop else 0
        for li in range(n_layers):
            P, (in_w, out_w, w1, w2), qkv, attn = _layer_qkv(h, params, li, dt)
            lse = torch.empty(B * nhead, T, device=h.device, dtype=torch.float32)
            _attention_fwd(qkv, attn, lse, T, B, nhead, dh, sep, (site_seed(drop[0], li, 0), thr) if thr else None)
            z1, mean1, rstd1, h1, u, u_is_grad, g, z2, mean2, rstd2, h2 = _layer_tail(h, attn, P, out_w, w1, w2, drop, li)
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
        flat, grads = _flat_grads(dev, *(p.shape for p in params))
        end = flat.numel()
        dh2 = dout.contiguous().to(dt)
        for li in reversed(range(n_layers)):
            P, G = _layer(params, li), _layer(grads, li)
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
            _attention_bwd(qkv, attn, lse, dattn, dqkv, delta, T, B, nhead, dh, sep,
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
            n = sum(t.numel() for t in G.values())     # this layer's 12 gradients are one contiguous slice of the flat buffer
            _bucket_ready(flat[end - n:end], wait=False)
            end -= n
        if GRAD_BUCKET_SYNC is not None:
            GRAD_BUCKET_SYNC()
        ctx.saved_acts = None
        return (dh2, None, None, None, None, None, None, None) + tuple(grads)


@torch.no_grad()
def encode_context(src, T, B, nhead, precision, *params, n_keys=None):
    """The K/V cache of T training rows: src [T*B, E] (their embedding, activation dtype, T >= 1) runs through the encoder
    layers with sep = T, and kv [n_layers, T*B, 2E] keeps each layer's K | V of those rows, as the in-projection produced
    them.  The last layer's attention and MLP are not run: no later layer reads their output.
    n_keys (int32 [B] on the device, optional): dataset b has n_keys[b] training rows; in the attention its row i attends
    to rows [0, n_keys[b]) and, when i >= n_keys[b] (a padding row), to itself."""
    dt, n_layers, dh, h = _stack_start(src, precision, nhead, params)
    N, E = h.shape
    kv = torch.empty(n_layers, N, 2 * E, device=src.device, dtype=dt)
    for li in range(n_layers):
        P, (_, out_w, w1, w2), qkv, attn = _layer_qkv(h, params, li, dt)
        kv[li].copy_(qkv[:, E:])
        if li == n_layers - 1:
            break
        if n_keys is None:
            lse = torch.empty(B * nhead, T, device=h.device, dtype=torch.float32)
            L.attention_fwd(qkv, attn, lse, T, B, nhead, dh, T)
        else:
            LR.attention_ragged_fwd(qkv, attn, T, B, nhead, dh, n_keys)
        h = _layer_tail(h, attn, P, out_w, w1, w2, None, li)[-1]
    return kv


@torch.no_grad()
def query_stack(src, kv, n, B, nhead, precision, *params, n_keys=None):
    """src [m*B, E] (the query rows' embedding, activation dtype) -> their output of the encoder layers, each query row
    attending to the n training rows whose K | V the cache kv [n_layers, n*B, 2E] holds (encode_context) and to itself:
    rows n .. n + m - 1 of EncoderStackFn on (training rows, query rows) with sep = n.  Per layer: the in-projection GEMM,
    the context attention, then the same out-projection, LayerNorm and MLP kernels as EncoderStackFn.forward.
    n_keys (int32 [B] on the device, optional): the query rows of dataset b attend to its first n_keys[b] cached rows only."""
    dt, n_layers, dh, h = _stack_start(src, precision, nhead, params, kv)
    for li in range(n_layers):
        P, (_, out_w, w1, w2), qkv, attn = _layer_qkv(h, params, li, dt)
        if n_keys is None:
            L.attention_ctx_fwd(qkv, kv[li], attn, h.shape[0] // B, n, B, nhead, dh)
        else:
            LR.attention_ctx_ragged_fwd(qkv, kv[li], attn, h.shape[0] // B, n, B, nhead, dh, n_keys)
        h = _layer_tail(h, attn, P, out_w, w1, w2, None, li)[-1]
    return h


class QueryStackFn(torch.autograd.Function):
    """query_stack with a backward to its input only: src [m*B, E] -> the query rows' output of the encoder layers against
    the cache kv.  The cache and every parameter are constants here: the backward runs the dgrad chain of each layer
    (LayerNorm, MLP, out-projection, context attention, in-projection) and forms no weight or bias gradient, so a
    parameter's .grad is left as it was.  The forward runs the kernels of query_stack, the context attention in its
    variant that also writes lse, so its output is query_stack's bit for bit."""

    @staticmethod
    def forward(ctx, src, kv, n, B, nhead, precision, n_keys, *params):
        dt, n_layers, dh, h = _stack_start(src, precision, nhead, params, kv)
        m = h.shape[0] // B
        saved = []
        for li in range(n_layers):
            P, (in_w, out_w, w1, w2), qkv, attn = _layer_qkv(h, params, li, dt)
            lse = torch.empty(B * nhead, m, device=h.device, dtype=torch.float32)
            LIG.attention_ctx_grad_fwd(qkv, kv[li], attn, lse, m, n, B, nhead, dh, n_keys)
            z1, mean1, rstd1, h1, u, u_is_grad, g, z2, mean2, rstd2, h2 = _layer_tail(h, attn, P, out_w, w1, w2, None, li)
            saved.append((qkv, attn, lse, z1, mean1, rstd1, u, z2, mean2, rstd2, in_w, out_w, w1, w2))
            h = h2
        ctx.saved_acts = saved
        ctx.u_is_grad = u_is_grad if n_layers else False
        ctx.params = params
        ctx.meta = (kv, n, B, nhead, precision, n_keys)
        return h

    @staticmethod
    def backward(ctx, dout):
        if ctx.saved_acts is None:
            raise RuntimeError("QueryStackFn: activations were already released by a previous backward "
                               "(retain_graph=True is not supported)")
        kv, n, B, nhead, precision, n_keys = ctx.meta
        dh2 = dout.contiguous().to(act_dtype(precision))
        N, E = dh2.shape
        m, dh = N // B, E // nhead
        for li in reversed(range(len(ctx.saved_acts))):
            P = _layer(ctx.params, li)
            qkv, attn, lse, z1, mean1, rstd1, u, z2, mean2, rstd2, in_w, out_w, w1, w2 = ctx.saved_acts[li]
            ctx.saved_acts[li] = None
            dz2 = torch.empty_like(z2)
            L.layernorm_bwd(dh2, z2, mean2, rstd2, P["g2"], dz2, None, None)
            du = _gelu_linear_dgrad(dz2, w2, u, ctx.u_is_grad)
            dh1 = _linear_dgrad(du, w1, aux=dz2)
            del dz2, du, u, z2
            dz1 = torch.empty_like(z1)
            L.layernorm_bwd(dh1, z1, mean1, rstd1, P["g1"], dz1, None, None)
            dattn = _linear_dgrad(dz1, out_w)
            del dh1, z1
            dqkv = torch.empty_like(qkv)
            delta = torch.empty_like(lse)
            LIG.attention_ctx_bwd(qkv, kv[li], attn, lse, dattn, dqkv, delta, m, n, B, nhead, dh, n_keys)
            del dattn, attn, qkv
            dh2 = _linear_dgrad(dqkv, in_w, aux=dz1)
            del dqkv, dz1
        ctx.saved_acts = None
        return (dh2,) + (None,) * (6 + len(ctx.params))


class EmbedFn(torch.autograd.Function):
    """(x [T,B,F], y [T,B]) -> src [T*B, E]:  x Wx^T + bx + (t < sep)(y wy + by)   (reference transformer.py:68-74);
    with a RaggedSeps `sep`, (t < n_keys[b]) for dataset b.  The backward returns the gradients of x (every row) and y
    (the rows with the y embedding, zero elsewhere) when they are asked for, and of the weights when those are."""

    @staticmethod
    def forward(ctx, x, y, Wx, bx, wy, by, sep, precision):
        L.require_cuda(x, y, Wx, bx, wy, by)
        T, B, F = x.shape
        E = Wx.shape[0]
        x = x.detach().contiguous().float()
        y_shape = y.shape
        y = y.detach().contiguous().float()
        out = torch.empty(T * B, E, device=x.device, dtype=act_dtype(precision))
        args = (x, y, Wx.detach().contiguous(), bx.detach().contiguous(), wy.detach().contiguous().view(-1),
                by.detach().contiguous(), out, T, B, F, E)
        if isinstance(sep, RaggedSeps):
            LRT.embed_ragged_fwd(*args, sep.n_keys)
        else:
            L.embed_fwd(*args, sep)
        ctx.save_for_backward(x, y, args[2], args[4])
        ctx.meta = (T, B, F, E, sep, wy.shape, y_shape)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, y, Wx, wy = ctx.saved_tensors
        T, B, F, E, sep, wy_shape, y_shape = ctx.meta
        dev = dout.device
        dout = dout.contiguous()
        ragged = isinstance(sep, RaggedSeps)
        dx = dy = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            dx = torch.empty(T, B, F, device=dev)
            dy = torch.empty(T * B, device=dev)
            LIG.embed_input_bwd(dout, Wx, wy, dx, dy, T, B, F, E, sep.s_max if ragged else sep,
                                sep.n_keys if ragged else None)
            dx = dx if ctx.needs_input_grad[0] else None
            dy = dy.view(y_shape) if ctx.needs_input_grad[1] else None
        if not any(ctx.needs_input_grad[2:6]):
            return dx, dy, None, None, None, None, None, None
        dWx = torch.zeros(E, F, device=dev)
        dbx = torch.zeros(E, device=dev)
        dwy = torch.zeros(E, device=dev)
        dby = torch.zeros(E, device=dev)
        if ragged:
            LRT.embed_ragged_bwd(dout, x, y, dWx, dbx, dwy, dby, T, B, F, E, sep.n_keys)
        else:
            L.embed_bwd(dout, x, y, dWx, dbx, dwy, dby, T, B, F, E, sep)
        return dx, dy, dWx, dbx, dwy.view(wy_shape), dby, None, None


def _f32_rows(rows, n, dev):
    """An uninitialised fp32 [rows, n] view whose row pitch is n rounded up to 4 (16-byte rows for the GEMM's stores)."""
    return torch.empty(rows, (n + 3) // 4 * 4, device=dev, dtype=torch.float32)[:, :n]


def _head_fwd(hq, w0, b0, w2, b2):
    """The two GEMMs every decoder head runs: g = GELU(hq w0^T + b0), then z = g w2^T + b2 into padded fp32 rows.
    Returns (g, u, u_is_grad, z) with u, u_is_grad as from _gelu_linear_fwd."""
    g, u, u_is_grad = _gelu_linear_fwd(hq, w0, b0)
    z = _f32_rows(hq.shape[0], w2.shape[0], hq.device)
    L.gemm(g, w2, z, bias=b2.detach().contiguous())
    return g, u, u_is_grad, z


def _head_bwd(dz, hq, u, g, u_is_grad, w0, w2, grads):
    """The backward of _head_fwd from dz = dL/dz (activation dtype): fills grads = (dW0, db0, dW2, db2) and returns
    dL/dhq."""
    dW0, db0, dW2, db2 = grads
    L.colsum(dz, db2)
    _linear_wgrad(dz, g, dW2)
    du = _gelu_linear_dgrad(dz, w2, u, u_is_grad)
    L.colsum(du, db0)
    _linear_wgrad(du, hq, dW0)
    return _linear_dgrad(du, w0)


def _head_dgrad(dz, u, u_is_grad, w0, w2):
    """dL/dhq of _head_fwd with its weights held constant (a head called with frozen parameters): the two dgrad GEMMs of
    _head_bwd alone, no weight gradient and no gradient bucket."""
    return _linear_dgrad(_gelu_linear_dgrad(dz, w2, u, u_is_grad), w0)


class DecoderFn(torch.autograd.Function):
    """hq [Nq, E] -> logits [Nq, n_out] fp32:  GELU(hq W0^T + b0) W2^T + b2  (reference transformer.py:23,85),
    applied to the query rows only (the reference computes all T rows and slices, transformer.py:91)."""

    @staticmethod
    def forward(ctx, hq, W0, b0, W2, b2, precision):
        L.require_cuda(hq, W0, b0, W2, b2)
        dt = act_dtype(precision)
        hq = hq.contiguous()
        w0, w2 = _cast(W0, dt), _cast(W2, dt)
        g, u, u_is_grad, logits = _head_fwd(hq, w0, b0, w2, b2)
        ctx.save_for_backward(hq, u, g, W0, W2, w0, w2)
        ctx.u_is_grad = u_is_grad
        ctx.precision = precision
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        hq, u, g, W0, W2, w0, w2 = ctx.saved_tensors
        dev = dlogits.device
        Nq, n_out = dlogits.shape
        dl = torch.zeros(Nq, (n_out + 7) // 8 * 8, device=dev, dtype=act_dtype(ctx.precision))
        dl[:, :n_out] = dlogits
        if not any(ctx.needs_input_grad[1:5]):
            return (_head_dgrad(dl[:, :n_out], u, ctx.u_is_grad, w0, w2),) + (None,) * 5
        flat, grads = _flat_grads(dev, W0.shape, W0.shape[:1], W2.shape, W2.shape[:1])
        dhq = _head_bwd(dl[:, :n_out], hq, u, g, ctx.u_is_grad, w0, w2, grads)
        _bucket_ready(flat)
        return (dhq, *grads, None)


def _head_grad_rows(dout, n_cols, dt):
    """The fp32 output gradient with unit column stride, and an uninitialised [Nq, n_cols rounded up to 8] buffer in the
    activation dtype for the row kernel to fill (the padding keeps the GEMM operands' row pitch a multiple of 16 bytes)."""
    dout = dout.float()
    if dout.stride(1) != 1:
        dout = dout.contiguous()
    return dout, torch.empty(dout.shape[0], (n_cols + 7) // 8 * 8, device=dout.device, dtype=dt)


class ScaledDecoderFn(torch.autograd.Function):
    """hq [Nq, E] -> (logits [Nq, n_out] fp32, temp [Nq] fp32) of decoders.ScaledDecoder (reference decoders.py:13-20):
    x = GELU(hq W^T + b); [z | zt] = x [W1; W2]^T + [b1; b2] in one GEMM against the stacked second-layer weights;
    temp = softmax(zt) . c and logits = z / temp in one row kernel (csrc/scaled_head.cu).  temp is not differentiable."""

    @staticmethod
    def forward(ctx, hq, W, b, W1, b1, W2, b2, precision):
        L.require_cuda(hq, W, b, W1, b1, W2, b2)
        dt = act_dtype(precision)
        hq = hq.contiguous()
        Nq, n_out = hq.shape[0], W1.shape[0]
        w = _cast(W, dt)
        w12 = torch.cat([W1.detach(), W2.detach()], 0).to(dt)
        b12 = torch.cat([b1.detach(), b2.detach()], 0).float()
        g, u, u_is_grad, zz = _head_fwd(hq, w, b, w12, b12)
        logits = _f32_rows(Nq, n_out, hq.device)
        temp = torch.empty(Nq, device=hq.device, dtype=torch.float32)
        L.scaled_head_fwd(zz, n_out, logits, temp)
        ctx.save_for_backward(hq, u, g, zz, temp, w, w12)
        ctx.mark_non_differentiable(temp)
        ctx.u_is_grad = u_is_grad
        ctx.meta = (precision, W.shape, W1.shape, W2.shape)
        return logits, temp

    @staticmethod
    def backward(ctx, dlogits, _dtemp):
        hq, u, g, zz, temp, w, w12 = ctx.saved_tensors
        precision, w_shape, w1_shape, w2_shape = ctx.meta
        n_out, nhid = w1_shape
        nz = n_out + L.HEAD_TEMPS
        dlogits, dzz = _head_grad_rows(dlogits, nz, act_dtype(precision))
        L.scaled_head_bwd(dlogits, zz, temp, n_out, dzz, dzz.shape[1])
        if not any(ctx.needs_input_grad[1:7]):
            return (_head_dgrad(dzz[:, :nz], u, ctx.u_is_grad, w, w12),) + (None,) * 7
        # [W1; W2] and [b1; b2] are contiguous in the bucket, so the stacked GEMM writes both layers' gradients in place
        flat, grads = _flat_grads(hq.device, w_shape, w_shape[:1], (nz, nhid), (nz,))
        dhq = _head_bwd(dzz[:, :nz], hq, u, g, ctx.u_is_grad, w, w12, grads)
        _bucket_ready(flat)
        dW, db, dW12, db12 = grads
        return dhq, dW, db, dW12[:n_out], db12[:n_out], dW12[n_out:], db12[n_out:], None


class FixedScaledDecoderFn(torch.autograd.Function):
    """hq [Nq, E] -> logits [Nq, n_out] fp32 of decoders.FixedScaledDecoder (reference decoders.py:22-30):
    (GELU(hq W0^T + b0) W2^T + b2) / sum(T).  The sum is formed on the device inside the row kernel; T's gradient is
    -sum(dlogits * z) / sum(T)^2 in every entry."""

    @staticmethod
    def forward(ctx, hq, W0, b0, W2, b2, T, precision):
        L.require_cuda(hq, W0, b0, W2, b2, T)
        dt = act_dtype(precision)
        hq = hq.contiguous()
        Nq, n_out = hq.shape[0], W2.shape[0]
        w0, w2 = _cast(W0, dt), _cast(W2, dt)
        g, u, u_is_grad, z = _head_fwd(hq, w0, b0, w2, b2)
        logits = _f32_rows(Nq, n_out, hq.device)
        S = torch.empty(1, device=hq.device, dtype=torch.float32)
        L.fixed_scaled_head_fwd(z, n_out, T.detach().contiguous().float(), logits, S)
        ctx.save_for_backward(hq, u, g, z, S, w0, w2)
        ctx.u_is_grad = u_is_grad
        ctx.meta = (precision, W0.shape, W2.shape, T.shape)
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        hq, u, g, z, S, w0, w2 = ctx.saved_tensors
        precision, w0_shape, w2_shape, t_shape = ctx.meta
        n_out = w2_shape[0]
        dlogits, dz = _head_grad_rows(dlogits, n_out, act_dtype(precision))
        frozen = not any(ctx.needs_input_grad[1:6])
        flat, grads = _flat_grads(hq.device, *((t_shape,) if frozen else (w0_shape, w0_shape[:1], w2_shape, w2_shape[:1],
                                                                          t_shape)))
        L.fixed_scaled_head_bwd(dlogits, z, S, n_out, dz, grads[-1], dz.shape[1])
        if frozen:
            return (_head_dgrad(dz[:, :n_out], u, ctx.u_is_grad, w0, w2),) + (None,) * 6
        dhq = _head_bwd(dz[:, :n_out], hq, u, g, ctx.u_is_grad, w0, w2, grads[:4])
        _bucket_ready(flat)
        return (dhq, *grads, None)


def conv_weight_operand(W, dgrad=False):
    """bf16 B operand of the 64 -> 64 tensor-core conv kernels: [64, 9, 64] (co, tap, ci) for the forward; for the data
    gradient (ci, tap, co) holding W[co, ci, 2 - dr, 2 - dc] at tap 3 dr + dc (the flipped kernel)."""
    W = W.detach()
    if dgrad:
        W = W.flip(2, 3).permute(1, 0, 2, 3)
    return W.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)


class ConvEncoderFn(torch.autograd.Function):
    """x [N, S*S] fp32 images -> [N, E] fp32: the conv stack of encoders.Conv (n_conv valid 3x3 convolutions + ReLU, the
    spatial mean, Linear(64, E)).  params: (weight, bias) of each applied conv, then the linear's weight and bias.
    Activations are NHWC in the activation dtype; each conv's post-ReLU output is kept for the backward (its own ReLU mask
    and the next layer's weight-gradient operand).  Gradient grids are zero-padded by 2 pixels; the kernels that produce
    them write the border too.  No gradient flows to x.  Every gradient is summed in a fixed order."""

    @staticmethod
    def forward(ctx, x, S, precision, keep, *params):
        L.require_cuda(x, *params)
        dt = act_dtype(precision)
        N = x.shape[0]
        convs, (lin_w, lin_b) = [params[i:i + 2] for i in range(0, len(params) - 2, 2)], params[-2:]
        h, s = x.detach().contiguous().float(), S
        acts = []
        for li, (W, b) in enumerate(convs):
            y = torch.empty(N, s - 2, s - 2, L.CONV_CH, device=x.device, dtype=dt)
            cin = 1 if li == 0 else L.CONV_CH
            w_op = conv_weight_operand(W) if (cin == L.CONV_CH and dt == torch.bfloat16) else W.detach().contiguous()
            L.conv_fwd(h, w_op, b.detach().contiguous(), y, N, s, cin)
            acts.append(y)
            h, s = y, s - 2
        feat = torch.empty(N, L.CONV_CH, device=x.device, dtype=dt)
        L.conv_mean_fwd(h, feat, N, s)
        lin_wc = _cast(lin_w, dt)
        out = _linear_fwd(feat, lin_wc, lin_b.detach().contiguous(), out_dtype=torch.float32)
        if keep and any(ctx.needs_input_grad):
            ctx.saved = (x.detach().contiguous().float(), acts, feat, lin_wc)
        else:
            ctx.saved = None
        ctx.meta = (S, precision)
        ctx.params = params
        return out

    @staticmethod
    def backward(ctx, dout):
        if ctx.saved is None:
            raise RuntimeError("ConvEncoderFn: no activations were kept (forward under no_grad, or a second backward)")
        x, acts, feat, lin_wc = ctx.saved
        ctx.saved = None
        S, precision = ctx.meta
        params = ctx.params
        dt = act_dtype(precision)
        dev = dout.device
        N, E = dout.shape
        dy = dout.contiguous().to(dt)
        # the projection's weight and bias gradients as ONE GEMM over [feat, 1] without split-K: a single store per
        # element, so that every gradient of the encoder is reproducible bit for bit (K = N images is short)
        feat1 = torch.zeros(N, L.CONV_CH + 8, device=dev, dtype=dt)
        feat1[:, :L.CONV_CH] = feat
        feat1[:, L.CONV_CH] = 1
        d_lin = torch.empty(E, L.CONV_CH + 8, device=dev)
        L.gemm(dy, feat1, d_lin, a_mn_major=True, b_mn_major=True, M=E, N=L.CONV_CH + 8, K=N)
        d_lin_w, d_lin_b = d_lin[:, :L.CONV_CH], d_lin[:, L.CONV_CH]
        dfeat = _linear_dgrad(dy, lin_wc)
        del dy, feat, feat1
        s = S - 2 * len(acts)
        g = torch.empty(N, s + 4, s + 4, L.CONV_CH, device=dev, dtype=dt)
        L.conv_mean_bwd(dfeat, acts[-1], g, N, s)
        grads = []
        for li in reversed(range(len(acts))):
            W = params[2 * li]
            s_in = s + 2
            cin = 1 if li == 0 else L.CONV_CH
            x_in = x if li == 0 else acts[li - 1]
            dW = torch.empty_like(W, dtype=torch.float32)
            db = torch.empty(L.CONV_CH, device=dev)
            L.conv_wgrad(g, x_in, dW, db, N, s_in, cin)
            grads = [dW, db] + grads
            if li > 0:
                g_in = torch.empty(N, s_in + 4, s_in + 4, L.CONV_CH, device=dev, dtype=dt)
                w_op = conv_weight_operand(W, dgrad=True) if dt == torch.bfloat16 else W.detach().contiguous()
                L.conv_dgrad(g, w_op, x_in, g_in, N, s_in)
                g = g_in
            acts[li] = None
            s = s_in
        return (None, None, None, None) + tuple(grads) + (d_lin_w, d_lin_b)


def layer_params(layer):
    """The 12 parameter tensors of one nn.TransformerEncoderLayer in LAYER_PARAM_NAMES order."""
    return (layer.self_attn.in_proj_weight, layer.self_attn.in_proj_bias, layer.self_attn.out_proj.weight,
            layer.self_attn.out_proj.bias, layer.linear1.weight, layer.linear1.bias, layer.linear2.weight,
            layer.linear2.bias, layer.norm1.weight, layer.norm1.bias, layer.norm2.weight, layer.norm2.bias)
