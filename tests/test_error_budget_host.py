"""The error bounds of oracle/error_budget.py on CPU restatements that round where the kernels round: a correct
restatement lies inside them at c = 1, and each numerical slip a kernel could make falls outside them at the constant
the GPU tests use.  Each perturbation also reports whether the max-scaled tolerances the GPU tests used before pass it."""
import math

import pytest
import torch

from oracle import error_budget as EB, pfn_oracle as O

BLK = 64


def _bf16(x):
    return x.to(torch.bfloat16).double()


def _qkv(T, B, H, dh, seed, q_scale=1.0, v_offset=0.0):
    g = torch.Generator().manual_seed(seed)
    E = H * dh
    x = torch.randn(T * B, 3 * E, generator=g, dtype=torch.float64)
    x[:, :E] *= q_scale
    x[:, 2 * E:] += v_offset
    return _bf16(x)


def flash_fwd(qkv, T, B, H, dh, sep, *, drop_diag=False, lazy_rescale=False, skip_block=None, lse_shift=0.0):
    """The tensor-core forward's algorithm: a row >= sep starts from its diagonal key (m = s_ii, l = 1, O = v_i), then
    64-key blocks of the train keys with an online softmax; P is rounded to bf16 before P V, O / l to bf16 at the end."""
    E = H * dh
    q, k, v = (EB._heads(qkv[:, n * E:(n + 1) * E], T, B, H, dh) for n in range(3))
    scale = 1.0 / math.sqrt(dh)
    diag = (torch.arange(T) >= sep) & (not drop_diag)
    s_ii = (q * k).sum(-1) * scale
    m = torch.where(diag, s_ii, torch.full_like(s_ii, float("-inf")))
    l = diag.double().expand_as(m).clone()
    o = v * diag.double().view(T, 1)
    for kb in range((sep + BLK - 1) // BLK):
        if kb == skip_block:
            continue
        j0, j1 = kb * BLK, min(sep, kb * BLK + BLK)
        s = q @ k[:, :, j0:j1].transpose(-1, -2) * scale
        mn = torch.maximum(m, s.amax(-1))
        corr = torch.exp(m - mn)
        p = torch.exp(s - mn.unsqueeze(-1))
        l = l * corr + p.sum(-1)
        o_corr = torch.where(corr > 0.98, torch.ones_like(corr), corr) if lazy_rescale else corr
        o = o * o_corr.unsqueeze(-1) + _bf16(p) @ v[:, :, j0:j1]
        m = mn
    out = _bf16(o / l.unsqueeze(-1))
    return EB._tokens(out, T, B, H, dh), (m + torch.log(l) + lse_shift).reshape(B * H, T)


def gemm_splitk(A, B, k_splits, *, drop_kblock=None, bf16_partials=False):
    """fp32 accumulation per 64-wide k-block, k_splits partial sums reduce-added into an fp32 output."""
    K = A.shape[1]
    nkb = (K + BLK - 1) // BLK
    C = torch.zeros(A.shape[0], B.shape[0], dtype=torch.float32)
    per = (nkb + k_splits - 1) // k_splits
    for sp in range(k_splits):
        acc = torch.zeros_like(C)
        for kb in range(sp * per, min(nkb, (sp + 1) * per)):
            if kb == drop_kblock:
                continue
            sl = slice(kb * BLK, min(K, kb * BLK + BLK))
            acc += A[:, sl].float() @ B[:, sl].float().t()
        C += acc.to(torch.bfloat16).float() if bf16_partials else acc
    return C


def _old_fwd_pass(out, lse, f):
    """The max-scaled forward tolerances the GPU tests used before the per-element bounds."""
    ok_out = (out - f["out"]).abs().max().item() <= 2e-2 * f["out"].abs().max().item()
    ok_lse = (lse - f["lse"]).abs().max().item() <= 2e-3 * (f["lse"].abs().max().item() + 1)
    return ok_out and ok_lse


def _ratio(got, exact, bound):
    return ((got - exact).abs() / bound).max().item()


# T, B, H, dh, sep: ragged T and sep, a diagonal-only problem, several key blocks
FWD_CASES = [(200, 2, 2, 128, 100), (300, 1, 2, 128, 299), (130, 1, 1, 128, 0), (256, 1, 2, 64, 256)]


@pytest.mark.parametrize("T,B,H,dh,sep", FWD_CASES)
def test_flash_restatement_inside_bound_at_c1(T, B, H, dh, sep):
    qkv = _qkv(T, B, H, dh, T + sep, q_scale=1.5)
    out, lse = flash_fwd(qkv, T, B, H, dh, sep)
    f = EB.attention_fwd(qkv, T, B, H, dh, sep, EB.U)
    EB.check_attention_fwd(out, lse, f, 1.0, 1.0)


def test_gemm_restatement_inside_bound_at_c1():
    g = torch.Generator().manual_seed(3)
    M, N, K = 64, 96, 64 * 200
    A, B = _bf16(torch.randn(M, K, generator=g)), _bf16(torch.randn(N, K, generator=g))
    exact, bound, _ = EB.gemm(A, B, EB.U32, EB.C_ACC_TC)
    EB.check("host split-K gemm fp32 out", gemm_splitk(A, B, 16), exact, bound, 1.0)
    C = gemm_splitk(A, B, 1).to(torch.bfloat16)
    exact, bound, _ = EB.gemm(A, B, EB.U, EB.C_ACC_TC)
    EB.check("host gemm bf16 out", C, exact, bound, 1.0)


# Each perturbation: (name, qkv builder, T, B, H, dh, sep, flash_fwd keyword, whether the old max-scaled tolerance passes it)
PERTURBATIONS = [
    # the diagonal key of the rows >= sep left out (the producer warps' job in the dQ kernel, folded in first here)
    ("drop_diagonal", dict(q_scale=1.5), 320, 2, 2, 128, 256, dict(drop_diag=True), False),
    # O not rescaled when the running max moves by less than ~2 %: keys whose scores rise slowly block by block
    ("lazy_rescale", "rising", 512, 1, 1, 128, 512, dict(lazy_rescale=True), False),
    ("lse_shift_1e-4", dict(q_scale=0.5), 200, 2, 2, 128, 150, dict(lse_shift=1e-4), True),
    ("skip_key_block", dict(q_scale=1.5), 300, 2, 2, 128, 260, dict(skip_block=2), False),
]


@pytest.mark.parametrize("name,data,T,B,H,dh,sep,kw,old_passes", PERTURBATIONS, ids=[p[0] for p in PERTURBATIONS])
def test_attention_perturbation_outside_bound(name, data, T, B, H, dh, sep, kw, old_passes):
    qkv = EB.rising_max_qkv(T, B, H, dh, torch.Generator().manual_seed(5)).double() if data == "rising" else _qkv(T, B, H, dh, 17 + T, **data)
    f = EB.attention_fwd(qkv, T, B, H, dh, sep, EB.U)
    clean_out, clean_lse = flash_fwd(qkv, T, B, H, dh, sep)
    assert _ratio(clean_out, f["out"], f["out_bound"]) <= 1.0 and _ratio(clean_lse, f["lse"], f["lse_bound"]) <= 1.0
    out, lse = flash_fwd(qkv, T, B, H, dh, sep, **kw)
    r_out, r_lse = _ratio(out, f["out"], f["out_bound"]), _ratio(lse, f["lse"], f["lse_bound"])
    old = _old_fwd_pass(out, lse, f)
    print(f"[perturbation] {name}: out err/bound {r_out:.3g} (c {EB.C_ATT_OUT}), lse err/bound {r_lse:.3g} "
          f"(c {EB.C_ATT_LSE}); old max-scaled tolerance {'PASSES' if old else 'fails'}")
    assert r_out > EB.C_ATT_OUT or r_lse > EB.C_ATT_LSE, f"{name} is inside the bound"
    assert old == old_passes, f"{name}: the old tolerance {'passes' if old else 'fails'} it"


# the wgrad shape of tests/test_gpu_gemm.py (K = 64 * 200, 16 splits) with fewer output rows: a dropped k-block, and each
# split's partial sum stored in bf16 before the fp32 reduce-add; old: 2e-3 max|C|
@pytest.mark.parametrize("name,kw,old_passes", [("drop_kblock", dict(drop_kblock=77), False),
                                                ("bf16_partials", dict(bf16_partials=True), True)])
def test_splitk_perturbation_outside_bound(name, kw, old_passes):
    g = torch.Generator().manual_seed(4)
    M, N, K = 64, 96, 64 * 200
    A, B = _bf16(torch.randn(M, K, generator=g)), _bf16(torch.randn(N, K, generator=g))
    exact, bound, _ = EB.gemm(A, B, EB.U32, EB.C_ACC_TC)
    C = gemm_splitk(A, B, 16, **kw).double()
    r = _ratio(C, exact, bound)
    old = (C - exact).abs().max().item() <= 2e-3 * exact.abs().max().item()
    print(f"[perturbation] splitk_{name}: err/bound {r:.3g} (c {EB.C_GEMM}); "
          f"old max-scaled tolerance {'PASSES' if old else 'fails'}")
    assert r > EB.C_GEMM
    assert old == old_passes


@pytest.mark.parametrize("T,B,H,dh,sep,p", [(40, 2, 2, 16, 17, 0.0), (33, 1, 3, 8, 0, 0.0), (30, 2, 1, 16, 30, 0.0),
                                            (24, 2, 2, 8, 11, 0.3)])
def test_exact_attention_matches_autograd(T, B, H, dh, sep, p):
    """The helpers' closed-form forward and backward are the derivative of the dense-mask attention (with the given
    dropout keep mask), and out_kernel = out_exact leaves no inherited delta term."""
    g = torch.Generator().manual_seed(T + sep)
    E = H * dh
    qkv = torch.randn(T * B, 3 * E, generator=g, dtype=torch.float64, requires_grad=True)
    dout = torch.randn(T * B, E, generator=g, dtype=torch.float64)
    keep = (torch.rand(B, H, T, T, generator=g) >= p).double() if p else None
    scale = 1.0 / (1.0 - p)
    heads = lambda t: EB._heads(t, T, B, H, dh)
    s = heads(qkv[:, :E]) @ heads(qkv[:, E:2 * E]).transpose(-1, -2) / math.sqrt(dh) + O.d_q_mask(T, T - sep, torch.float64)
    P = torch.softmax(s, -1)
    ref = EB._tokens((P if keep is None else P * keep * scale) @ heads(qkv[:, 2 * E:]), T, B, H, dh)
    (ref * dout).sum().backward()
    f = EB.attention_fwd(qkv.detach(), T, B, H, dh, sep, EB.U, keep, scale)
    assert torch.allclose(f["out"], ref.detach(), atol=1e-12)
    assert torch.allclose(f["lse"], torch.logsumexp(s, -1).reshape(B * H, T).detach(), atol=1e-12)
    b = EB.attention_bwd(f, dout, f["out"])
    for n, name in enumerate(("dq", "dk", "dv")):
        assert torch.allclose(b[name], qkv.grad[:, n * E:(n + 1) * E], atol=1e-11), name
        assert (b[name + "_bound"] >= 0).all()


@pytest.mark.parametrize("K,req,want", [(640, 4, (4, 3)), (576, 4, (3, 3)), (64, 8, (1, 1)), (131072, 33, (33, 63)),
                                        (512000, 16, (16, 500)), (512000, 5, (5, 1600)), (256000, 33, (33, 122))])
def test_splitk_launch_normalises_the_request(K, req, want):
    """Nine k-blocks asked to split 4 ways take 3 per split and so launch 3 splits; the engine's full-size requests
    launch as asked."""
    assert EB.splitk_launch(K, req) == want
