"""The engine stage checks (oracle/engine_stages.py) on a CPU restatement of two bf16 encoder layers: the kernels are
restated in float32 with bf16 rounding where the engine stores, the layers' forward and backward call them the way
engine.EncoderStackFn does, and the calls are recorded and checked by the same code as the GPU test.  The correct
restatement stays inside every bound at c = 1; each wiring slip below falls outside its stage's bound at the GPU
constants.  Each slip also reports whether the end-to-end tolerances of the bf16 engine tests (gradient norms within
6 %, elements within 8 % of the tensor's largest gradient) pass it."""
import math
import types

import pytest
import torch

from oracle import engine_stages as ES, error_budget as EB

T, B, H, DH, NHID, SEP, NLAYERS = 24, 2, 2, 128, 512, 10, 2
E = H * DH
N = T * B
NUM_SMS = 132
THR = 51                     # p = 0.2
SEED = 1234567
BF = torch.bfloat16


def site_seed(seed, layer, site):
    return (int(seed) + 0x9E3779B9 * (4 * layer + site + 1)) & 0xFFFFFFFF


def keep_bits(seed, rows, cols, thr):
    """Counter-free stand-in for the kernels' masks: a keep byte per element drawn from the site's seed."""
    g = torch.Generator().manual_seed(int(seed))
    return (torch.randint(0, 256, (rows, cols), generator=g) >= thr).to(torch.uint8)


def _heads(t):
    return t.double().reshape(T, B, H, DH).permute(1, 2, 0, 3)


def _tokens(t):
    return t.permute(2, 0, 1, 3).reshape(N, E)


class FakeLib:
    """The kernels as float32 restatements with the kernels' signatures; bf16 rounding wherever they store bf16."""

    def __init__(self):
        self.noscale = False             # slip: dropout without 1 / (1 - p)
        self.rowdot_unrounded = False    # slip: ROWDOT from the fp32 accumulator instead of the stored bf16 C

    def gemm(self, A, B, C, *, a_mn_major=False, b_mn_major=False, bias=None, aux=None, C2=None, epilogue=0,
             accumulate=False, k_splits=1, M=None, N=None, K=None, use_tc=None, rowdot=None, c2_gelu_grad=False):
        Al = (A.t() if a_mn_major else A).double()
        Bl = (B.t() if b_mn_major else B).double()
        y = (Al @ Bl.t()).float()
        if bias is not None:
            y = y + bias.float()
        if epilogue == 1:
            if C2 is not None:
                C2.copy_((EB.gelu_grad(y.double()).float() if c2_gelu_grad else y).to(C2.dtype))
            y = torch.nn.functional.gelu(y)
        elif epilogue == 2:
            y = y * EB.gelu_grad(aux.double()).float()
        elif epilogue == 4:
            y = y * aux.float()
        elif epilogue == 3:
            c = y if self.rowdot_unrounded else y.to(C.dtype).float()
            rd, w = rowdot
            rd += (c.double() * aux.double()).reshape(y.shape[0], -1, w).sum(-1).float()
        elif aux is not None:
            y = y + aux.float()
        C.copy_((C.float() + y if accumulate else y).to(C.dtype))

    def _probs(self, qkv, drop):
        q, k, v = (_heads(qkv[:, n * E:(n + 1) * E]) for n in range(3))
        ok = EB.allowed_keys(T, SEP, "cpu")
        s = (q @ k.transpose(-1, -2) / math.sqrt(DH)).masked_fill(~ok, float("-inf"))
        P = torch.softmax(s, -1)
        km = torch.ones_like(P)
        if drop is not None:
            km = keep_bits(drop[0], B * H * T, T, drop[1]).double().reshape(B, H, T, T) * (256.0 / (256 - drop[1]))
        return q, k, v, s, P, km

    def attention_fwd(self, qkv, out, lse, T_, B_, H_, dh, sep, use_tc=None, batch_major=False, drop=None):
        q, k, v, s, P, km = self._probs(qkv, drop)
        out.copy_(_tokens((P * km) @ v).to(out.dtype))
        lse.copy_(torch.logsumexp(s, -1).reshape(B * H, T).float())

    def attention_bwd(self, qkv, out, lse, dout, dqkv, delta, T_, B_, H_, dh, sep, use_tc=None, batch_major=False,
                      drop=None, dq_colsum=None, delta_token_major=False):
        q, k, v, s, P, km = self._probs(qkv, drop)
        do = _heads(dout)
        if delta_token_major:
            dl = delta.double().reshape(T, B, H).permute(1, 2, 0).unsqueeze(-1)
        else:
            dl = (do * _heads(out)).sum(-1, keepdim=True)
            delta.copy_(dl.squeeze(-1).reshape(B * H, T).float())
        dS = P * ((do @ v.transpose(-1, -2)) * km - dl) / math.sqrt(DH)
        grads = (dS @ k, dS.transpose(-1, -2) @ q, (P * km).transpose(-1, -2) @ do)
        for n, g in enumerate(grads):
            dqkv[:, n * E:(n + 1) * E] = _tokens(g).to(dqkv.dtype)
        if dq_colsum is not None:
            dq_colsum += dqkv[:, :E].double().sum(0).float()

    def layernorm_fwd(self, z, gamma, beta, h, mean, rstd, eps=1e-5):
        zd = z.double()
        mu = zd.mean(-1, keepdim=True)
        r = 1.0 / torch.sqrt(((zd - mu) ** 2).mean(-1, keepdim=True) + eps)
        mean.copy_(mu.squeeze(-1).float())
        rstd.copy_(r.squeeze(-1).float())
        h.copy_(((zd - mean.double().unsqueeze(-1)) * rstd.double().unsqueeze(-1) * gamma.double() + beta.double()).to(h.dtype))

    def layernorm_bwd(self, dh, z, mean, rstd, gamma, dz, dgamma, dbeta, colsum_out=None):
        r = rstd.double().unsqueeze(-1)
        xh = (z.double() - mean.double().unsqueeze(-1)) * r
        dd = dh.double()
        g = dd * gamma.double()
        d = r * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
        dz.copy_(d.to(dz.dtype))
        dgamma += (dd * xh).sum(0).float()
        dbeta += dd.sum(0).float()
        if colsum_out is not None:
            colsum_out += d.sum(0).float()

    def colsum(self, X, out, N=None):
        out += X.double().sum(0).float()

    def dropout(self, x, out, seed, thr, residual=None):
        keep = keep_bits(seed, x.shape[0], x.shape[1], thr).float()
        sc = 1.0 if self.noscale else float(torch.tensor(256.0 / (256 - thr), dtype=torch.float32))
        y = x.float() * keep * sc
        if residual is not None:
            y = y + residual.float()
        out.copy_(y.to(out.dtype))

    def embed_fwd(self, *a, **k):
        raise NotImplementedError

    embed_bwd = bar_nll_fwd = bar_nll_bwd = embed_fwd


def _params(seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)
    layers = []
    for _ in range(NLAYERS):
        layers.append({"in_w": r(3 * E, E) * E ** -0.5, "in_b": r(3 * E) * 0.1, "out_w": r(E, E) * 0.5 * E ** -0.5,
                       "out_b": r(E) * 0.1, "w1": r(NHID, E) * E ** -0.5, "b1": r(NHID) * 0.1,
                       "w2": r(E, NHID) * 0.5 * NHID ** -0.5, "b2": r(E) * 0.1, "g1": 1 + 0.1 * r(E), "be1": 0.1 * r(E),
                       "g2": 1 + 0.1 * r(E), "be2": 0.1 * r(E)})
    return layers, r(N, E).to(BF), r(N, E).to(BF)


def stack_step(L, layers, src, dout, thr, slip=None):
    """engine.EncoderStackFn's forward and backward on the bf16 head-dim-128 path, with one optional wiring slip."""
    def lin(x, w, bias=None, aux=None, epi=0, C2=None, c2g=False, out_dtype=None):
        y = torch.empty(x.shape[0], w.shape[0], dtype=out_dtype or x.dtype)
        L.gemm(x, w, y, bias=bias, aux=aux, C2=C2, epilogue=epi, c2_gelu_grad=c2g)
        return y

    def dgrad(dy, w, aux=None, epi=0, rowdot=None):
        dx = torch.empty(dy.shape[0], w.shape[1], dtype=dy.dtype)
        L.gemm(dy, w, dx, b_mn_major=True, aux=aux, epilogue=epi, M=dy.shape[0], N=w.shape[1], K=w.shape[0], rowdot=rowdot)
        return dx

    def wgrad(dy, x, dw):
        L.gemm(dy, x, dw, a_mn_major=True, b_mn_major=True, accumulate=True, M=dw.shape[0], N=dw.shape[1], K=dy.shape[0])

    saved, h = [], src
    for li, P in enumerate(layers):
        wc = {k: P[k].to(BF) for k in ("in_w", "out_w", "w1", "w2")}
        qkv = lin(h, wc["in_w"], P["in_b"])
        attn = torch.empty(N, E, dtype=BF)
        lse = torch.empty(B * H, T)
        L.attention_fwd(qkv, attn, lse, T, B, H, DH, SEP, drop=(site_seed(SEED, li, 0), thr) if thr else None)
        if thr:
            z1 = lin(attn, wc["out_w"], P["out_b"])
            L.dropout(z1, z1, site_seed(SEED, li, 1), thr, residual=h)
        else:
            z1 = lin(attn, wc["out_w"], P["out_b"], aux=h)
        h1, m1, r1 = torch.empty_like(z1), torch.empty(N), torch.empty(N)
        L.layernorm_fwd(z1, P["g1"], P["be1"], h1, m1, r1)
        u = torch.empty(N, NHID, dtype=BF)
        g = lin(h1, wc["w1"], P["b1"], epi=1, C2=u, c2g=True)
        if thr:
            L.dropout(g, g, site_seed(SEED, li, 2), thr)
            z2 = lin(g, wc["w2"], P["b2"])
            L.dropout(z2, z2, site_seed(SEED, li, 3), thr, residual=h1)
        else:
            z2 = lin(g, wc["w2"], P["b2"], aux=h1)
        h2, m2, r2 = torch.empty_like(z2), torch.empty(N), torch.empty(N)
        L.layernorm_fwd(z2, P["g2"], P["be2"], h2, m2, r2)
        saved.append((h, qkv, attn, lse, z1, m1, r1, h1, u, g, z2, m2, r2, wc))
        h = h2
    out = h
    grads = [{k: torch.zeros_like(v) for k, v in P.items()} for P in layers]
    dh2 = dout
    for li in reversed(range(NLAYERS)):
        P, G = layers[li], grads[li]
        h, qkv, attn, lse, z1, m1, r1, h1, u, g, z2, m2, r2, wc = saved[li]
        if slip == "gelu_grad_other_layer":
            u = saved[1 - li][8]
        dz2 = torch.empty_like(z2)
        L.layernorm_bwd(dh2, z2, m2, r2, P["g2"], dz2, G["g2"], G["be2"],
                        G["b2"] if (not thr or slip == "b2_colsum_out_with_dropout") else None)
        L.noscale = slip == "bwd_mask_no_scale"
        dm = dz2
        if thr:
            dm = torch.empty_like(dz2)
            L.dropout(dz2, dm, site_seed(SEED, li, 2 if slip == "bwd_mask_site2" else 3), thr)
            L.colsum(dm, G["b2"])
        wgrad(dm, g, G["w2"])
        du = dgrad(dm, wc["w2"], aux=u, epi=4)
        if thr:
            L.dropout(du, du, site_seed(SEED, li, 2), thr)
        L.colsum(du, G["b1"])
        wgrad(du, h1, G["w1"])
        dh1 = dgrad(du, wc["w1"], aux=None if slip == "dh1_no_aux" else dz2)
        dz1 = torch.empty_like(z1)
        L.layernorm_bwd(dh1, z1, m1, r1, P["g1"], dz1, G["g1"], G["be1"], None if thr else G["out_b"])
        da = dz1
        if thr:
            da = torch.empty_like(dz1)
            L.dropout(dz1, da, site_seed(SEED, li, 1), thr)
            L.colsum(da, G["out_b"])
        L.noscale = False
        wgrad(da, attn, G["out_w"])
        delta = torch.zeros(N, H)
        dattn = dgrad(da, wc["out_w"], aux=attn, epi=3, rowdot=(delta, DH))
        dqkv = torch.empty_like(qkv)
        fused = not thr
        a_li = li + 1 if slip == "att_bwd_next_layer_seed" else li
        L.attention_bwd(qkv, attn, lse, dattn, dqkv, delta, T, B, H, DH, SEP,
                        drop=(site_seed(SEED, a_li, 0), thr) if thr else None,
                        dq_colsum=G["in_b"][:E] if fused else None, delta_token_major=True)
        if fused:
            W = P["out_w"]
            G["in_b"][2 * E:] += {"v_third_no_w": lambda: G["out_b"],
                                  "v_third_w_transposed": lambda: G["out_b"] @ W.t()}.get(slip, lambda: G["out_b"] @ W)()
        else:
            L.colsum(dqkv, G["in_b"])
        wgrad(dqkv, h, G["in_w"])
        dh2 = dgrad(dqkv, wc["in_w"], aux=dz1)
    return out, grads


def _run(thr, slip=None, c=None):
    layers, src, dout = _params(3)
    lib = FakeLib()
    lib.rowdot_unrounded = slip == "delta_unrounded"
    rec = ES.Recorder(lib).install()
    _, grads = stack_step(lib, layers, src, dout, thr, slip)
    rec.remove()
    mask = lambda li, site, rows, cols: keep_bits(site_seed(SEED, li, site), rows, cols, thr)
    chk = ES.StageCheck(T=T, B=B, H=H, sep=SEP, thr=thr, mask=mask, num_sms=NUM_SMS, c=c,
                        paths={"u_is_grad": True, "rowdot": True, "fused_bias": not thr}, tag=f"{slip or 'clean'}: ")
    return chk, rec.calls, layers, src, dout, grads


def _check(thr, slip=None, c=None):
    chk, calls, layers, src, dout, grads = _run(thr, slip, c)
    chk.stack(calls, layers, src, dout, grads)
    return chk, grads


@pytest.mark.parametrize("thr", [0, THR])
def test_restatement_inside_bounds_at_c1(thr):
    chk, _ = _check(thr, c=1.0)
    chk.report(f"restatement thr={thr}")
    assert max(chk.worst.values()) <= 1.0


def _old_tolerances_pass(grads, ref):
    """The bf16 engine tests' end-to-end tolerances: norms within 6 %, elements within 8 % of the tensor's largest."""
    for g, r in zip(grads, ref):
        for k in g:
            a, b = g[k].double(), r[k].double()
            if abs(a.norm() - b.norm()) > 6e-2 * b.norm() + 1e-5:
                return False
            if (a - b).abs().max() > 8e-2 * b.abs().max() + 1e-12:
                return False
    return True


SLIPS = [("bwd_mask_site2", THR, "dm"), ("att_bwd_next_layer_seed", THR, "dqkv"), ("bwd_mask_no_scale", THR, "dm"),
         ("b2_colsum_out_with_dropout", THR, "db2"), ("dh1_no_aux", 0, "dh1"), ("gelu_grad_other_layer", 0, "du"),
         ("v_third_no_w", 0, "din_b v"), ("v_third_w_transposed", 0, "din_b v"), ("delta_unrounded", 0, "delta")]


@pytest.mark.parametrize("slip,thr,stage", SLIPS)
def test_wiring_slip_falls_outside_its_stage(slip, thr, stage):
    _, ref = _check(thr)
    chk, calls, layers, src, dout, grads = _run(thr, slip)
    with pytest.raises(AssertionError) as e:
        chk.stack(calls, layers, src, dout, grads)
    assert f"{slip}: {stage}:" in str(e.value), str(e.value)
    print(f"[engine-stages host] {slip}: {str(e.value)[:160]}; old end-to-end tolerances "
          f"{'pass' if _old_tolerances_pass(grads, ref) else 'fail'} it")
