"""Op-by-op check of the engine's training step -- TEST INFRASTRUCTURE ONLY.

`Recorder` replaces the kernel entry points of a library namespace (`transformerscandobayesianinference_b200._lib`, or a
CPU restatement with the same signatures) with wrappers that keep every argument as it was before the call and every
buffer the call writes as it is after it.  `StageCheck` then walks the recorded calls of one step, asserts the call plan
of the engine path (the sequence of functions and the epilogue of every GEMM), and holds each stage to the per-element
bound of oracle/error_budget.py.

Each stage's exact fp64 value is computed from the engine's own stored outputs of earlier stages, chosen by their role
in the reference layer (torch `TransformerEncoderLayer`, oracle/pfn_oracle.encoder_layer_dropout_ref), never from the
pointers the engine handed the kernel.  Rounding therefore does not compound and every stage is held to its kernel's
own constant; a wrong tensor, mask, seed or missing term moves a stage's ratio by orders of magnitude.  Masks come from
`mask(layer, site, rows, cols)`, the keep bits the kernels regenerate (sites: 0 attention probabilities, 1 attention
block output, 2 after the GELU, 3 MLP block output).

The checks run on whatever device the records are on.
"""
import inspect

import torch

from . import error_budget as EB

LAYER_PARAM_NAMES = ("in_w", "in_b", "out_w", "out_b", "w1", "b1", "w2", "b2", "g1", "be1", "g2", "be2")
EPI_NAMES = {0: "none", 1: "gelu", 2: "gelu_bwd", 3: "rowdot", 4: "mul"}

# the arguments each recorded function writes (in place, accumulated or fresh)
OUTPUTS = {
    "gemm": ("C", "C2", "rowdot"),
    "attention_fwd": ("out", "lse"),
    "attention_bwd": ("dqkv", "delta", "dq_colsum"),
    "layernorm_fwd": ("h", "mean", "rstd"),
    "layernorm_bwd": ("dz", "dgamma", "dbeta", "colsum_out"),
    "colsum": ("out",),
    "dropout": ("out",),
    "embed_fwd": ("out",),
    "embed_bwd": ("dWx", "dbx", "dwy", "dby"),
    "bar_nll_fwd": ("nll", "idx", "lse", "oob_count"),
    "bar_nll_bwd": ("dlogits",),
}


def snap(t):
    """A copy of an argument.  A 2-D row-major view whose rows are padded keeps the padding columns (see `padded`)."""
    if isinstance(t, tuple):
        return tuple(snap(x) for x in t)
    if not torch.is_tensor(t):
        return t
    if t.dim() == 2 and t.shape[0] > 0 and t.stride(1) == 1 and t.stride(0) > t.shape[1]:
        ld = t.stride(0)
        if t.storage_offset() + t.shape[0] * ld <= t.untyped_storage().nbytes() // t.element_size():
            return t.as_strided((t.shape[0], ld), (ld, 1)).clone()[:, :t.shape[1]]
    return t.clone()


def padded(t):
    """The full rows (padding included) of a snapshot taken by `snap`."""
    return t.as_strided((t.shape[0], t.stride(0)), (t.stride(0), 1))


class Call:
    __slots__ = ("fn", "a", "out")

    def __init__(self, fn, a, out):
        self.fn, self.a, self.out = fn, a, out

    @property
    def sig(self):
        if self.fn != "gemm":
            return self.fn
        return "gemm/" + EPI_NAMES[int(self.a["epilogue"])] + ("/acc" if self.a["accumulate"] else "")


class Recorder:
    """Wraps the OUTPUTS entry points of `lib`: arguments before the call (`Call.a`), written buffers after (`Call.out`)."""

    def __init__(self, lib):
        self.lib = lib
        self.calls = []
        self._orig = {}

    def install(self):
        for name in OUTPUTS:
            real = getattr(self.lib, name)
            self._orig[name] = real
            setattr(self.lib, name, self._wrap(name, real))
        return self

    def remove(self):
        for name, real in self._orig.items():
            setattr(self.lib, name, real)
        self._orig = {}

    def _wrap(self, name, real):
        sig = inspect.signature(real)
        outs = OUTPUTS[name]

        def wrapper(*args, **kwargs):
            b = sig.bind(*args, **kwargs)
            b.apply_defaults()
            a = {k: snap(v) for k, v in b.arguments.items()}
            r = real(*args, **kwargs)
            self.calls.append(Call(name, a, {k: snap(b.arguments[k]) for k in outs if b.arguments.get(k) is not None}))
            return r
        return wrapper


def layer_plan(drop, u_is_grad, rowdot, fused_bias):
    """Per-layer call signatures of EncoderStackFn's forward and backward on one path."""
    fwd = (["gemm/none", "attention_fwd", "gemm/none"] + (["dropout"] if drop else []) + ["layernorm_fwd", "gemm/gelu"]
           + (["dropout", "gemm/none", "dropout"] if drop else ["gemm/none"]) + ["layernorm_fwd"])
    bwd = (["layernorm_bwd"] + (["dropout", "colsum"] if drop else [])
           + ["gemm/none/acc", "gemm/mul" if u_is_grad else "gemm/gelu_bwd"] + (["dropout"] if drop else [])
           + ["colsum", "gemm/none/acc", "gemm/none", "layernorm_bwd"] + (["dropout", "colsum"] if drop else [])
           + ["gemm/none/acc", "gemm/rowdot" if rowdot else "gemm/none", "attention_bwd"]
           + ([] if fused_bias else ["colsum"]) + ["gemm/none/acc", "gemm/none"])
    return fwd, bwd


def _u(t):
    return EB.U32 if t.dtype == torch.float32 else EB.U


def _expect(calls, plan, what):
    got = [c.sig for c in calls]
    assert got == plan, f"{what}: call plan {got} != expected {plan}"


class StageCheck:
    """Stage checks of one step.  mask(layer, site, rows, cols) -> 0/1 keep tensor; thr = 0: no dropout.  paths:
    u_is_grad (the forward stores GELU'), rowdot (delta from the out-projection dgrad), fused_bias (in-projection bias from
    dq_colsum and colsum(dz1) W_out).  c: one constant for every stage instead of the kernels' own (the CPU restatement
    passes at c = 1)."""

    def __init__(self, *, T, B, H, sep, thr, mask, num_sms, paths, c=None, tag=""):
        self.T, self.B, self.H, self.sep, self.thr, self.mask = T, B, H, sep, thr, mask
        self.num_sms, self.paths, self.c, self.tag = num_sms, paths, c, tag
        self.s = 256.0 / (256.0 - thr) if thr else 1.0
        self.worst = {}

    # ---------------------------------------------------------------- primitives
    def chk(self, stage, got, exact, bound, c):
        r = EB.check(f"{self.tag}{stage}", got, exact, bound, self.c if self.c is not None else c, verbose=False)
        self.worst[stage] = max(self.worst.get(stage, 0.0), r)

    def bitwise(self, stage, ok):
        assert bool(ok), f"{self.tag}{stage}: not bitwise equal to its exact value"
        self.worst.setdefault(stage, 0.0)

    def gemm(self, stage, c, A, Bm, *, bias=None, aux=None, epi="none", out="C"):
        """One GEMM launch: C = epi(A Bm^T + bias) (+ aux) with logical operands chosen by role."""
        got = c.out[out]
        tc = A.dtype == torch.bfloat16
        c_acc = (EB.C_ACC_WGRAD if c.a["accumulate"] else EB.C_ACC_TC) if tc else EB.C_ACC_SIMT
        ex, bd, _ = EB.gemm(A, Bm, _u(got), c_acc, bias=bias, aux=aux, epilogue=epi, fast_gelu=tc)
        self.chk(stage, got, ex, bd, EB.C_GEMM)
        return got

    def weight(self, stage, c, master):
        """The GEMM's weight operand must be the activation-dtype copy of the current fp32 master, bit for bit."""
        w = c.a["B"]
        self.bitwise(stage + " weight", w.dtype == c.a["A"].dtype and torch.equal(w, master.detach().to(w.dtype)))
        return w

    def dropout(self, stage, c, x, keep, residual=None):
        got = c.out["out"]
        ex, bd = EB.dropout(x, keep, self.thr, residual, _u(got))
        self.chk(stage, got, ex, bd, EB.C_DROPOUT)
        return got

    def colsum(self, stage, c, X):
        """A bias gradient: the column sums of X into a zeroed gradient buffer."""
        got = c.out["out"]
        depth = EB.colsum_depth(X.shape[0], X.shape[1], X.stride(0), X.element_size(), self.num_sms)
        ex, bd = EB.colsum(X, torch.zeros_like(got), depth)
        self.chk(stage, got, ex, bd, EB.C_ROWSUM)
        return got

    def ln_fwd(self, stage, c, z, gamma, beta):
        f = EB.layernorm_fwd(z, gamma, beta, _u(z))
        self.chk(stage, c.out["h"], f["h"], f["h_bound"], EB.C_LN)
        self.chk(stage + " mean", c.out["mean"], f["mean"], f["mean_bound"], EB.C_LN)
        self.chk(stage + " rstd", c.out["rstd"], f["rstd"], f["rstd_bound"], EB.C_LN)
        return c.out["h"], c.out["mean"], c.out["rstd"]

    def ln_bwd(self, stage, c, dh, z, gamma, mean, rstd, names):
        """LayerNorm backward into zeroed gamma / beta (/ bias, names[2]) gradients."""
        E = z.shape[1]
        depth = EB.ln_bwd_colsum_depth(z.shape[0], E, z.element_size(), EB.ln_vec(E, [E, E, E]), self.num_sms)
        b = EB.layernorm_bwd(dh, z, gamma, mean, rstd, _u(z), depth)
        self.chk(stage, c.out["dz"], b["dz"], b["dz_bound"], EB.C_LN_GRAD)
        self.chk(names[0], c.out["dgamma"], b["dgamma"], b["dgamma_bound"], EB.C_LN_GRAD)
        self.chk(names[1], c.out["dbeta"], b["dbeta"], b["dbeta_bound"], EB.C_LN_GRAD)
        if "colsum_out" in c.out:
            self.chk(names[2], c.out["colsum_out"], b["colsum"], b["colsum_bound"], EB.C_LN_GRAD)
        return c.out["dz"], b

    def keep(self, li, site, rows, cols):
        return self.mask(li, site, rows, cols) if self.thr else None

    # ---------------------------------------------------------------- one encoder layer
    def layer(self, li, fwd, bwd, p, x_in, dh_in, grads=None):
        """Forward and backward of layer li.  p: its fp32 master parameters by LAYER_PARAM_NAMES; x_in: its input as the
        engine stored it; dh_in: the gradient of its output as the engine handed it; grads: its final gradients (the
        in-projection bias is completed outside any kernel on the fused path)."""
        T, B, H, sep = self.T, self.B, self.H, self.sep
        drop = bool(self.thr)
        N, E = x_in.shape
        dh = E // H
        nhid = p["w1"].shape[0]
        pf, pb = layer_plan(drop, self.paths["u_is_grad"], self.paths["rowdot"], self.paths["fused_bias"])
        _expect(fwd, pf, f"layer {li} forward")
        _expect(bwd, pb, f"layer {li} backward")
        f, b = iter(fwd), iter(bwd)
        u_at = _u(x_in)
        k0 = self.keep(li, 0, B * H * T, T)
        k0 = None if k0 is None else k0.reshape(B, H, T, T)
        k1, k2, k3 = self.keep(li, 1, N, E), self.keep(li, 2, N, nhid), self.keep(li, 3, N, E)
        # ---- forward
        c = next(f)
        qkv = self.gemm("qkv", c, x_in, self.weight("qkv", c, p["in_w"]), bias=p["in_b"])
        c = next(f)
        fa = EB.attention_fwd(qkv, T, B, H, dh, sep, u_at, k0, self.s)
        self.chk("attn", c.out["out"], fa["out"], fa["out_bound"], EB.C_ATT_OUT)
        self.chk("lse", c.out["lse"], fa["lse"], fa["lse_bound"], EB.C_ATT_LSE)
        attn = c.out["out"]
        c = next(f)
        w_out = self.weight("z1", c, p["out_w"])
        if drop:
            z1 = self.dropout("z1", next(f), self.gemm("z1 pre", c, attn, w_out, bias=p["out_b"]), k1, x_in)
        else:
            z1 = self.gemm("z1", c, attn, w_out, bias=p["out_b"], aux=x_in)
        h1, mean1, rstd1 = self.ln_fwd("h1", next(f), z1, p["g1"], p["be1"])
        c = next(f)
        assert bool(c.a["c2_gelu_grad"]) == self.paths["u_is_grad"], f"layer {li}: GELU' path"
        w1 = self.weight("g", c, p["w1"])
        g = self.gemm("g", c, h1, w1, bias=p["b1"], epi="gelu")
        u = self.gemm("u", c, h1, w1, bias=p["b1"], epi="gelu_grad" if self.paths["u_is_grad"] else "none", out="C2")
        if drop:
            g = self.dropout("g", next(f), g, k2)
        c = next(f)
        w2 = self.weight("z2", c, p["w2"])
        if drop:
            z2 = self.dropout("z2", next(f), self.gemm("z2 pre", c, g, w2, bias=p["b2"]), k3, h1)
        else:
            z2 = self.gemm("z2", c, g, w2, bias=p["b2"], aux=h1)
        h2, mean2, rstd2 = self.ln_fwd("h2", next(f), z2, p["g2"], p["be2"])
        # ---- backward
        dz2, _ = self.ln_bwd("dz2", next(b), dh_in, z2, p["g2"], mean2, rstd2, ("dg2", "dbe2", "db2"))
        dm = dz2
        if drop:
            dm = self.dropout("dm", next(b), dz2, k3)
            self.colsum("db2", next(b), dm)
        self.gemm("dw2", next(b), dm.t(), g.t())
        c = next(b)
        du = self.gemm("du", c, dm, self.weight("du", c, p["w2"]).t(), aux=u,
                       epi="mul" if self.paths["u_is_grad"] else "gelu_bwd")
        if drop:
            du = self.dropout("du", next(b), du, k2)
        self.colsum("db1", next(b), du)
        self.gemm("dw1", next(b), du.t(), h1.t())
        c = next(b)
        dh1 = self.gemm("dh1", c, du, self.weight("dh1", c, p["w1"]).t(), aux=dz2)
        c_ln1 = next(b)
        dz1, lb1 = self.ln_bwd("dz1", c_ln1, dh1, z1, p["g1"], mean1, rstd1, ("dg1", "dbe1", "dout_b"))
        da = dz1
        if drop:
            da = self.dropout("da", next(b), dz1, k1)
            self.colsum("dout_b", next(b), da)
        self.gemm("dw_out", next(b), da.t(), attn.t())
        c = next(b)
        dattn = self.gemm("dattn", c, da, self.weight("dattn", c, p["out_w"]).t())
        delta = None
        if self.paths["rowdot"]:
            delta = c.out["rowdot"][0]
            ex, bd = EB.rowdot(dattn, attn, dh)
            self.chk("delta", delta, ex, bd, EB.C_ROWDOT)
        c = next(b)
        assert bool(c.a["delta_token_major"]) == self.paths["rowdot"], f"layer {li}: delta path"
        assert (c.a["dq_colsum"] is not None) == self.paths["fused_bias"], f"layer {li}: bias path"
        assert (c.a["drop"] is not None) == drop, f"layer {li}: attention dropout"
        bb = EB.attention_bwd(fa, dattn, attn, delta_kernel=delta)
        dqkv = c.out["dqkv"]
        for n, name in enumerate(("dq", "dk", "dv")):
            self.chk("dqkv", dqkv[:, n * E:(n + 1) * E], bb[name], bb[name + "_bound"], EB.C_ATT_GRAD)
        if self.paths["fused_bias"]:
            dq_sum = c.out["dq_colsum"]
            self.chk("din_b q", dq_sum, bb["dq"].sum(0), bb["dq_bound"].sum(0), EB.C_ATT_GRAD)
            if grads is not None:
                gb = grads["in_b"]
                self.bitwise("din_b q final", torch.equal(gb[:E], dq_sum))
                self.bitwise("din_b k", bool((gb[E:2 * E] == 0).all()))
                bound = EB.bias_v_fused(dattn, da, p["out_w"], c_ln1.out["colsum_out"], lb1, EB.C_ACC_TC)
                self.chk("din_b v", gb[2 * E:], bb["dv"].sum(0), bound, EB.C_BIAS_FUSED)
        else:
            self.colsum("din_b", next(b), dqkv)
        self.gemm("dw_in", next(b), dqkv.t(), x_in.t())
        c = next(b)
        dh_out = self.gemm("dh", c, dqkv, self.weight("dh", c, p["in_w"]).t(), aux=dz1)
        return h2, dh_out

    # ---------------------------------------------------------------- the encoder stack
    def stack(self, calls, layers, x_in, dh_top, grads=None):
        """calls: the stack's forward (layer 0 first) then its backward (last layer first); layers: per-layer parameter
        dicts; x_in: the stack's input as stored; dh_top: the gradient handed to the stack.  The records of a layer are
        dropped once it is checked.  Returns (h_out, dh_in) of the stack."""
        n = len(layers)
        pf, pb = layer_plan(bool(self.thr), self.paths["u_is_grad"], self.paths["rowdot"], self.paths["fused_bias"])
        nf, nb = len(pf), len(pb)
        assert len(calls) == n * (nf + nb), f"stack: {len(calls)} calls for {n} layers of {nf} + {nb}"
        fwd = [calls[i * nf:(i + 1) * nf] for i in range(n)]
        bwd = [calls[n * nf + (n - 1 - i) * nb:n * nf + (n - i) * nb] for i in range(n)]
        calls.clear()
        h, dh0 = x_in, None
        for li in range(n):
            dh_in = dh_top if li == n - 1 else bwd[li + 1][-1].out["C"]
            h, dh = self.layer(li, fwd[li], bwd[li], layers[li], h, dh_in, None if grads is None else grads[li])
            if li == 0:
                dh0 = dh
            fwd[li] = bwd[li] = None
        return h, dh0

    # ---------------------------------------------------------------- one training step
    def step(self, calls, *, x, y, emb, layers, dec, precision, borders=None, full_support=True, grads=None):
        """embedding -> layers -> decoder -> loss (bar head when borders is given; otherwise the loss is not a kernel)
        -> backward.  x [T, B, F], y [T, B]; emb = (Wx, bx, wy, by), dec = (W0, b0, W2, b2) fp32 masters."""
        T, B, sep = self.T, self.B, self.sep
        N, nq = T * B, (T - sep) * B
        dt = torch.bfloat16 if precision == "bf16" else torch.float32
        n = len(layers)
        pf, pb = layer_plan(bool(self.thr), self.paths["u_is_grad"], self.paths["rowdot"], self.paths["fused_bias"])
        bar = borders is not None
        dg = "gemm/mul" if self.paths["u_is_grad"] else "gemm/gelu_bwd"
        head = ["gemm/gelu", "gemm/none"] + (["bar_nll_fwd", "bar_nll_bwd"] if bar else [])
        dec_b = ["colsum", "gemm/none/acc", dg, "colsum", "gemm/none/acc", "gemm/none"]
        sig = [c.sig for c in calls]
        want = ["embed_fwd"] + pf * n + head + dec_b + pb * n + ["embed_bwd"]
        assert sig == want, f"step: call plan {sig} != expected {want}"
        Wx, bx, wy, by = emb
        W0, b0, W2, b2 = dec
        F = x.shape[-1]
        x2, y1 = x.reshape(N, F), y.reshape(N)
        # embedding
        c_ef = calls[0]
        ex, bd = EB.embed_fwd(x2, y1, Wx, bx, wy, by, sep * B, _u(c_ef.out["out"]))
        self.chk("embed", c_ef.out["out"], ex, bd, EB.C_EMBED)
        x_in = c_ef.out["out"]
        i = 1 + n * len(pf)
        stack_fwd = calls[1:i]
        # decoder on the query rows of the last layer's output (its stored h2)
        h_last = stack_fwd[-1].out["h"]
        hq = h_last[sep * B:]
        c = calls[i]
        w0 = self.weight("dec g", c, W0)
        g_dec = self.gemm("dec g", c, hq, w0, bias=b0, epi="gelu")
        u_dec = self.gemm("dec u", c, hq, w0, bias=b0, epi="gelu_grad" if self.paths["u_is_grad"] else "none", out="C2")
        c = calls[i + 1]
        logits = self.gemm("logits", c, g_dec, self.weight("logits", c, W2), bias=b2)
        i += 2
        dl = None
        if bar:
            c_nf, c_nb = calls[i], calls[i + 1]
            n_out = logits.shape[1]
            self.bitwise("loss logits", torch.equal(c_nf.a["logits"].reshape(nq, n_out), logits))
            fb = EB.bar_nll_fwd(logits, y[sep:].reshape(nq), borders, full_support)
            self.chk("nll", c_nf.out["nll"], fb["nll"], fb["nll_bound"], EB.C_BAR)
            self.chk("loss lse", c_nf.out["lse"], fb["lse"], fb["lse_bound"], EB.C_BAR)
            self.bitwise("loss idx", torch.equal(c_nb.a["idx"], c_nf.out["idx"]))
            ex, bd = EB.bar_nll_bwd(logits, c_nf.out["idx"], c_nf.out["lse"], c_nb.a["g"], EB.U32)
            dl = c_nb.out["dlogits"]
            self.chk("dlogits", dl, ex, bd, EB.C_BAR_GRAD)
            i += 2
        # decoder backward: dl is the activation-dtype copy of dlogits, its padding columns zero
        c = calls[i]
        dlv = c.a["X"]
        n_out = dlv.shape[1]
        if dl is not None:
            self.bitwise("dl", torch.equal(dlv, dl.reshape(nq, n_out).to(dt)))
        self.bitwise("dl padding", bool((padded(dlv)[:, n_out:] == 0).all()))
        self.colsum("dec db2", c, dlv)
        self.gemm("dec dW2", calls[i + 1], dlv.t(), g_dec.t())
        c = calls[i + 2]
        du = self.gemm("dec du", c, dlv, self.weight("dec du", c, W2).t(), aux=u_dec,
                       epi="mul" if self.paths["u_is_grad"] else "gelu_bwd")
        self.colsum("dec db0", calls[i + 3], du)
        self.gemm("dec dW0", calls[i + 4], du.t(), hq.t())
        c = calls[i + 5]
        dhq = self.gemm("dhq", c, du, self.weight("dhq", c, W0).t())
        i += 6
        # the stack receives dhq on the query rows and exact zeros on the train rows (slice backward of hq)
        dh_top = torch.zeros(N, dhq.shape[1], dtype=dt, device=dhq.device)
        dh_top[sep * B:] = dhq
        self.bitwise("dh stack", torch.equal(calls[i].a["dh"], dh_top))
        c_eb = calls[-1]
        stack = stack_fwd + calls[i:-1]
        del calls[:]
        _, dh0 = self.stack(stack, layers, x_in, dh_top, grads)
        eb = EB.embed_bwd(dh0, x2, y1, sep * B, EB.embed_bwd_depth(N))
        for name in ("dWx", "dbx", "dwy", "dby"):
            got = c_eb.out[name]
            self.chk("embed " + name, got, eb[name][0].reshape(got.shape), eb[name][1].reshape(got.shape), EB.C_ROWSUM)

    def report(self, what):
        for stage, r in self.worst.items():
            print(f"[engine-stages] {what} {stage}: worst err/bound = {r:.4g}")
