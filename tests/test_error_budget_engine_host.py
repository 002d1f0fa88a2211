"""The engine stage checks (oracle/engine_stages.py) on the CPU: engine.EncoderStackFn runs two bf16 encoder layers
forward and backward through a float32 fake of the kernel library (the kernels restated with bf16 rounding where they
store bf16), and the calls are recorded and checked by the same code as the GPU test.  The engine stays inside every
bound at c = 1; each wiring slip below, made by the fake at the one library call it concerns, falls outside its stage's
bound at the GPU constants.  The forward alone, run under torch.no_grad() as inference runs it, is checked the same way
with its own slips.  Each slip also reports whether the end-to-end tolerances of the bf16 engine tests
(gradient norms within 6 %, elements within 8 % of the tensor's largest gradient) pass it."""
import math

import pytest
import torch

from oracle import engine_stages as ES, error_budget as EB
from transformerscandobayesianinference_b200 import _lib, engine

T, B, H, DH, NHID, SEP, NLAYERS = 24, 2, 2, 128, 512, 10, 2
E = H * DH
N = T * B
NUM_SMS = 132
THR = 51                     # p = 0.2
SEED = 1234567
BF = torch.bfloat16
SITES = {engine.site_seed(SEED, li, site): (li, site) for li in range(NLAYERS) for site in range(4)}


def keep_bits(seed, rows, cols, thr):
    """Counter-free stand-in for the kernels' masks: a keep byte per element drawn from the site's seed."""
    g = torch.Generator().manual_seed(int(seed))
    return (torch.randint(0, 256, (rows, cols), generator=g) >= thr).to(torch.uint8)


class FakeLib:
    """What the engine reads of the kernel library: the kernels as float32 restatements with the kernels' signatures and
    bf16 rounding wherever they store bf16, and the bf16 tensor-core path taken everywhere.  `slip` names one wiring
    mistake, which the fake makes at the call it concerns."""
    EPI_NONE, EPI_GELU, EPI_GELU_BWD, EPI_ROWDOT, EPI_MUL = (_lib.EPI_NONE, _lib.EPI_GELU, _lib.EPI_GELU_BWD,
                                                             _lib.EPI_ROWDOT, _lib.EPI_MUL)

    def __init__(self, slip=None):
        self.slip = slip
        self.backward = False     # the stack's backward has begun (its first call is a layernorm_bwd)
        self.ln_bwd_calls = 0     # the backward of each layer calls layernorm_bwd for LN2, then for LN1
        self.dz2 = None           # dz of the latest LN2 backward
        self.b2_extra = None      # LN2's column sum of dz under dropout, for the next colsum
        self.gelu_grads = []      # C2 of the forward's gemm/gelu calls, one per layer

    def require_cuda(self, *tensors):
        pass

    def num_sms(self, device=None):
        return NUM_SMS

    def tc_gemm_ok(self, *args):
        return True

    def tc_attention_ok(self, *args):
        return True

    def gemm(self, A, B, C, *, a_mn_major=False, b_mn_major=False, bias=None, aux=None, C2=None, epilogue=EPI_NONE,
             accumulate=False, k_splits=1, M=None, N=None, K=None, use_tc=None, rowdot=None, c2_gelu_grad=False):
        if epilogue == self.EPI_GELU:
            self.gelu_grads.append(C2)
            if self.slip == "g_stale_weight":
                # the bf16 copy of W1 from before ten Adam steps of lr 1e-3: every element 1e-2 away from the current one
                step = torch.randn(B.shape, generator=torch.Generator().manual_seed(5)).sign()
                B = (B.float() + 1e-2 * step).to(B.dtype)
        elif epilogue == self.EPI_MUL and self.slip == "gelu_grad_other_layer":
            aux = next(u for u in self.gelu_grads if u is not aux)
        if self.slip == "dh1_no_aux" and aux is not None and aux is self.dz2:
            aux = None
        Al = (A.t() if a_mn_major else A).double()
        Bl = (B.t() if b_mn_major else B).double()
        if accumulate and self.slip == "wgrad_lost_token":
            Al, Bl = Al[:, :-1], Bl[:, :-1]
        y = (Al @ Bl.t()).float()
        if bias is not None:
            y = y + bias.float()
        if epilogue == self.EPI_GELU:
            if C2 is not None:
                C2.copy_((EB.gelu_grad(y.double()).float() if c2_gelu_grad else y).to(C2.dtype))
            y = torch.nn.functional.gelu(y)
        elif epilogue == self.EPI_GELU_BWD:
            y = y * EB.gelu_grad(aux.double()).float()
        elif epilogue == self.EPI_MUL:
            y = y * aux.float()
        elif epilogue == self.EPI_ROWDOT:
            c = y if self.slip == "delta_unrounded" else y.to(C.dtype).float()
            rd, w = rowdot
            rd += (c.double() * aux.double()).reshape(y.shape[0], -1, w).sum(-1).float()
        elif aux is not None:
            y = y + aux.float()
        C.copy_((C.float() + y if accumulate else y).to(C.dtype))

    def _probs(self, qkv, drop, sep=SEP):
        q, k, v = (EB._heads(qkv[:, n * E:(n + 1) * E].double(), T, B, H, DH) for n in range(3))
        ok = EB.allowed_keys(T, sep, "cpu")
        s = (q @ k.transpose(-1, -2) / math.sqrt(DH)).masked_fill(~ok, float("-inf"))
        P = torch.softmax(s, -1)
        km = torch.ones_like(P)
        if drop is not None:
            km = keep_bits(drop[0], B * H * T, T, drop[1]).double().reshape(B, H, T, T) * (256.0 / (256 - drop[1]))
        return q, k, v, s, P, km

    def attention_fwd(self, qkv, out, lse, T, B, H, dh, sep, use_tc=None, batch_major=False, drop=None):
        # attn_sep_plus_1: the first query row is taken for a train row, so every later query row sees it as a key
        q, k, v, s, P, km = self._probs(qkv, drop, sep + 1 if self.slip == "attn_sep_plus_1" else sep)
        out.copy_(EB._tokens((P * km) @ v, T, B, H, dh).to(out.dtype))
        lse.copy_(torch.logsumexp(s, -1).reshape(B * H, T).float())

    def attention_bwd(self, qkv, out, lse, dout, dqkv, delta, T, B, H, dh, sep, use_tc=None, batch_major=False,
                      drop=None, dq_colsum=None, delta_token_major=False):
        if self.slip == "att_bwd_next_layer_seed" and drop is not None:
            drop = (engine.site_seed(SEED, SITES[drop[0]][0] + 1, 0), drop[1])
        q, k, v, s, P, km = self._probs(qkv, drop)
        do = EB._heads(dout.double(), T, B, H, dh)
        if delta_token_major:
            dl = delta.double().reshape(T, B, H).permute(1, 2, 0).unsqueeze(-1)
        else:
            dl = (do * EB._heads(out.double(), T, B, H, dh)).sum(-1, keepdim=True)
            delta.copy_(dl.squeeze(-1).reshape(B * H, T).float())
        dS = P * ((do @ v.transpose(-1, -2)) * km - dl) / math.sqrt(DH)
        grads = (dS @ k, dS.transpose(-1, -2) @ q, (P * km).transpose(-1, -2) @ do)
        for n, g in enumerate(grads):
            dqkv[:, n * E:(n + 1) * E] = EB._tokens(g, T, B, H, dh).to(dqkv.dtype)
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
        self.backward = True
        ln2 = self.ln_bwd_calls % 2 == 0
        self.ln_bwd_calls += 1
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
        if ln2:
            self.dz2 = dz
            if self.slip == "b2_colsum_out_with_dropout" and colsum_out is None:
                self.b2_extra = d.sum(0).float()

    def colsum(self, X, out, N=None):
        out += X.double().sum(0).float()
        if self.b2_extra is not None:
            out += self.b2_extra
            self.b2_extra = None

    def dropout(self, x, out, seed, thr, residual=None):
        if self.slip == "bwd_mask_site2" and self.backward and SITES[seed][1] == 3:
            seed = engine.site_seed(SEED, SITES[seed][0], 2)
        keep = keep_bits(seed, x.shape[0], x.shape[1], thr).float()
        noscale = self.backward and self.slip == "bwd_mask_no_scale"
        sc = 1.0 if noscale else float(torch.tensor(256.0 / (256 - thr), dtype=torch.float32))
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


def _step(lib, layers, src, dout, thr, slip=None):
    """engine.EncoderStackFn's forward and backward on `lib` (delta and GELU' fusions on); the layers' gradients.  The
    v third of the in-projection bias gradient is formed outside the library, so its slips are made here."""
    names = engine.LAYER_PARAM_NAMES
    params = [P[k].detach().requires_grad_() for P in layers for k in names]
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(engine, "L", lib)
        mp.setattr(engine, "_DELTA_FUSION", True)
        mp.setattr(engine, "_GELU_GRAD_FWD", True)
        out = engine.EncoderStackFn.apply(src, T, B, SEP, H, "bf16", True, (SEED, thr) if thr else None, *params)
        out.backward(dout)
    grads = [dict(zip(names, (p.grad for p in params[i:i + len(names)]))) for i in range(0, len(params), len(names))]
    for P, G in zip(layers, grads):
        if slip == "v_third_no_w":
            G["in_b"][2 * E:] = G["out_b"]
        elif slip == "v_third_w_transposed":
            G["in_b"][2 * E:] = G["out_b"] @ P["out_w"].t()
    return grads


def _run(thr, slip=None, c=None):
    layers, src, dout = _params(3)
    lib = FakeLib(slip)
    rec = ES.Recorder(lib).install()
    grads = _step(lib, layers, src, dout, thr, slip)
    rec.remove()
    mask = lambda li, site, rows, cols: keep_bits(engine.site_seed(SEED, li, site), rows, cols, thr)
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
    chk.report(f"engine thr={thr}")
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
# slips of the forward alone, caught in the training step as well as in an inference forward
FWD_SLIPS = [("attn_sep_plus_1", "attn"), ("g_stale_weight", "g")]
SLIPS += [(slip, 0, stage) for slip, stage in FWD_SLIPS]


@pytest.mark.parametrize("slip,thr,stage", SLIPS)
def test_wiring_slip_falls_outside_its_stage(slip, thr, stage):
    _, ref = _check(thr)
    chk, calls, layers, src, dout, grads = _run(thr, slip)
    with pytest.raises(AssertionError) as e:
        chk.stack(calls, layers, src, dout, grads)
    assert f"{slip}: {stage}:" in str(e.value), str(e.value)
    print(f"[engine-stages host] {slip}: {str(e.value)[:160]}; old end-to-end tolerances "
          f"{'pass' if _old_tolerances_pass(grads, ref) else 'fail'} it")


# ---------------------------------------------------------------------------------------------------------------------
# The forward alone, as inference runs it (the tabular evaluation): EncoderStackFn under torch.no_grad() keeps no
# activation, and StageCheck.stack_fwd checks its calls
# ---------------------------------------------------------------------------------------------------------------------
def _forward(slip=None, c=None):
    layers, src, _ = _params(3)
    lib = FakeLib(slip)
    rec = ES.Recorder(lib).install()
    params = [P[k] for P in layers for k in engine.LAYER_PARAM_NAMES]
    with pytest.MonkeyPatch.context() as mp, torch.no_grad():
        mp.setattr(engine, "L", lib)
        mp.setattr(engine, "_GELU_GRAD_FWD", True)
        out = engine.EncoderStackFn.apply(src, T, B, SEP, H, "bf16", torch.is_grad_enabled(), None, *params)
    rec.remove()
    assert out.grad_fn is None
    chk = ES.StageCheck(T=T, B=B, H=H, sep=SEP, thr=0, mask=None, num_sms=NUM_SMS, c=c,
                        paths={"u_is_grad": True, "rowdot": True, "fused_bias": True}, tag=f"{slip or 'clean'}: ")
    return chk, rec.calls, layers, src, out


def test_forward_restatement_inside_bounds_at_c1():
    chk, calls, layers, src, out = _forward(c=1.0)
    pf, _ = ES.layer_plan(False, True, True, True)
    assert [c.sig for c in calls] == pf * NLAYERS
    h = chk.stack_fwd(calls, layers, src)
    assert torch.equal(h, out)
    chk.report("engine forward")
    assert set(chk.worst) == {"qkv", "qkv weight", "attn", "lse", "z1", "z1 weight", "h1", "h1 mean", "h1 rstd", "g",
                              "g weight", "u", "z2", "z2 weight", "h2", "h2 mean", "h2 rstd"}
    assert max(chk.worst.values()) <= 1.0


@pytest.mark.parametrize("slip,stage", FWD_SLIPS)
def test_forward_slip_falls_outside_its_stage(slip, stage):
    chk, calls, layers, src, _ = _forward(slip)
    with pytest.raises(AssertionError) as e:
        chk.stack_fwd(calls, layers, src)
    assert f"{slip}: {stage}:" in str(e.value), str(e.value)
    print(f"[engine-stages host] forward {slip}: {str(e.value)[:160]}")


# ---------------------------------------------------------------------------------------------------------------------
# ES.ReductionCheck, the inline checker of the full-size steps, on the same engine run: its wrappers assert the call plan
# as the calls are made and check the token-axis reductions from the calls' own operands, 7 rows at a time (a block that
# does not divide the 48 tokens)
# ---------------------------------------------------------------------------------------------------------------------
def _reductions(thr, slip=None, c=None):
    layers, src, dout = _params(3)
    lib = FakeLib(slip)
    chk = ES.ReductionCheck(lib, n_layers=NLAYERS, drop=bool(thr), head=None, num_sms=NUM_SMS, block=7, c=c,
                            paths={"u_is_grad": True, "rowdot": True, "fused_bias": not thr},
                            splits=engine._wgrad_splits, tag=f"{slip or 'clean'}: ").install()
    try:
        grads = _step(lib, layers, src, dout, thr, slip)
    finally:
        chk.remove()
    chk.finish(layers, grads)
    return chk


@pytest.mark.parametrize("thr", [0, THR])
def test_reduction_check_restatement_inside_bounds_at_c1(thr):
    chk = _reductions(thr, c=1.0)
    chk.report(f"engine thr={thr}")
    want = {"dw2", "dw1", "dw_out", "dw_in", "dg2", "dbe2", "db2", "db1", "dg1", "dbe1", "dout_b"}
    want |= {"din_b"} if thr else {"din_b q", "din_b q final", "din_b k", "din_b v"}
    assert set(chk.worst) == want
    assert max(chk.worst.values()) <= 1.0
    assert chk.k_splits == {s: {1} for s in ("dw2", "dw1", "dw_out", "dw_in")}


@pytest.mark.parametrize("slip,thr,stage", [("wgrad_lost_token", 0, "dw2"), ("v_third_no_w", 0, "din_b v"),
                                            ("b2_colsum_out_with_dropout", THR, "db2")])
def test_reduction_check_catches_slip(slip, thr, stage):
    """A weight gradient short of one token, a v third without W_out, and a bias gradient summed twice (LN2's column sum
    of dz under dropout added into the b2 gradient as well as the colsum after the mask)."""
    with pytest.raises(AssertionError) as e:
        _reductions(thr, slip)
    assert f"{slip}: {stage}" in str(e.value), str(e.value)


def test_reduction_check_asserts_the_plan_as_it_runs():
    """A path the step does not take (the delta from a separate pass instead of the out-projection dgrad) fails at the
    first call that differs, while the step runs."""
    layers, src, dout = _params(3)
    lib = FakeLib()
    chk = ES.ReductionCheck(lib, n_layers=NLAYERS, drop=False, head=None, num_sms=NUM_SMS, splits=engine._wgrad_splits,
                            paths={"u_is_grad": True, "rowdot": False, "fused_bias": True}).install()
    try:
        with pytest.raises(AssertionError, match="is gemm/rowdot where the plan has gemm/none"):
            _step(lib, layers, src, dout, 0)
    finally:
        chk.remove()
