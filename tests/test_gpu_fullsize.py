"""Full-size checks at BASELINE.json's headline configuration (cfg 2: T=1000, E=512, 6 layers, nhid 1024, 4 heads, 100 bars,
sep=500, batch 512) through size-independent properties and sub-sampled oracle comparisons -- the dense oracle cannot run
the whole problem in seconds, but it can run a few (batch, head) slices / rows of it.

Everything goes through the C ABI (`_lib`) or the public modules on top of it."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from transformerscandobayesianinference_b200 import _lib as L, bar_distribution, encoders, priors, transformer
from oracle import error_budget as EB, pfn_oracle as O

T, B, F, E, H, NHID, NL, NB, SEP = 1000, 512, 1, 512, 4, 1024, 6, 100, 500
DH = E // H


def test_attention_fullsize_slices_match_oracle(cuda_device):
    """tensor-core attention fwd+bwd on the full [T*B, 3E] tensor; three (batch, head) slices re-done by the dense-mask oracle."""
    torch.manual_seed(11)
    qkv = torch.randn(T * B, 3 * E, device=cuda_device).to(torch.bfloat16)
    out = torch.empty(T * B, E, device=cuda_device, dtype=torch.bfloat16)
    lse = torch.empty(B * H, T, device=cuda_device)
    L.attention_fwd(qkv, out, lse, T, B, H, DH, SEP, use_tc=True)
    dout = torch.randn(T * B, E, device=cuda_device).to(torch.bfloat16)
    dqkv = torch.full_like(qkv, float("nan"))
    delta = torch.empty_like(lse)
    L.attention_bwd(qkv, out, lse, dout, dqkv, delta, T, B, H, DH, SEP, use_tc=True)
    assert torch.isfinite(out.float()).all() and torch.isfinite(dqkv.float()).all()
    q3 = qkv.view(T, B, 3, H, DH)
    for (b, h) in [(0, 0), (257, 2), (511, 3)]:
        one = q3[:, b, :, h, :].reshape(T, 3 * DH)                                 # a 1-batch 1-head problem
        f = EB.attention_fwd(one, T, 1, 1, DH, SEP, EB.U)
        got = out.view(T, B, H, DH)[:, b, h, :]
        EB.check_attention_fwd(got, lse[b * H + h].view(1, T), f, EB.C_ATT_OUT, EB.C_ATT_LSE)
        do = dout.view(T, B, H, DH)[:, b, h, :]
        gd = dqkv.view(T, B, 3, H, DH)[:, b, :, h, :].reshape(T, 3 * DH)
        EB.check_attention_bwd(gd, EB.attention_bwd(f, do, got), EB.C_ATT_GRAD)


def test_gemm_fullsize_rows_match_reference(cuda_device):
    """512000 x 1536 x 512 projection (wgmma path): random output rows against fp64 dot products."""
    torch.manual_seed(12)
    N = T * B
    x = torch.randn(N, E, device=cuda_device).to(torch.bfloat16)
    w = (torch.randn(3 * E, E, device=cuda_device) / E ** 0.5).to(torch.bfloat16)
    bias = torch.randn(3 * E, device=cuda_device)
    y = torch.empty(N, 3 * E, device=cuda_device, dtype=torch.bfloat16)
    L.gemm(x, w, y, bias=bias, use_tc=True)
    rows = torch.tensor([0, 1, 127, 128, 255, 256, 65537, 300001, N - 129, N - 1], device=cuda_device)
    ref, bound, _ = EB.gemm(x[rows], w, EB.U, EB.C_ACC_TC, bias=bias)
    EB.check("gemm fullsize rows", y[rows], ref, bound, EB.C_GEMM)
    # linearity in the rows: the GEMM of a row-permuted input is the row-permuted output, bit for bit
    perm = torch.randperm(N, device=cuda_device)
    y2 = torch.empty_like(y)
    L.gemm(x[perm].contiguous(), w, y2, bias=bias, use_tc=True)
    assert torch.equal(y2, y[perm])


def _model(dev):
    torch.manual_seed(13)
    m = transformer.TransformerModel(encoders.Linear(F, E), NB, E, H, NHID, NL, 0.0, y_encoder=encoders.Linear(1, E)).to(dev)
    # the reference zero-initialises out_proj / linear2 (transformer.py:43-53): give them weight so every path matters
    with torch.no_grad():
        for layer in m.transformer_encoder.layers:
            layer.self_attn.out_proj.weight.normal_(0, E ** -0.5)
            layer.linear2.weight.normal_(0, NHID ** -0.5)
    return m.eval()


def test_model_fullsize_mask_and_batch_properties(cuda_device):
    """Forward of the full cfg-2 model: (i) datasets are independent: permuting the batch permutes the logits bit for bit;
    (ii) the single_eval_pos mask: a query row's logits do not change when OTHER query rows change, and they do not see
    the query targets y[sep:] at all; (iii) they DO depend on the training set."""
    dev = cuda_device
    model = _model(dev)
    x, y, _ = priors.fast_gp.get_batch(B, T, F, device=str(dev), hyperparameters={"noise": 1e-4, "outputscale": 1., "lengthscale": .6})
    with torch.no_grad():
        base = model((x, y), single_eval_pos=SEP)                       # [T-sep, B, NB]
        assert base.shape == (T - SEP, B, NB) and torch.isfinite(base.float()).all()
        perm = torch.randperm(B, device=dev)
        assert torch.equal(model((x[:, perm], y[:, perm]), single_eval_pos=SEP), base[:, perm])
        y2 = y.clone(); y2[SEP:] = torch.randn_like(y2[SEP:])            # query targets are never an input
        assert torch.equal(model((x, y2), single_eval_pos=SEP), base)
        x3 = x.clone(); x3[SEP + 7] += 1.0                                # another query row moves ...
        out3 = model((x3, y), single_eval_pos=SEP)
        keep = torch.ones(T - SEP, dtype=torch.bool, device=dev); keep[7] = False
        assert torch.equal(out3[keep], base[keep])                        # ... nobody else notices
        assert not torch.equal(out3[7], base[7])
        y4 = y.clone(); y4[:SEP] += 0.5                                   # the training targets matter to every query row
        assert (model((x, y4), single_eval_pos=SEP).float() - base.float()).abs().amax(dim=(1, 2)).min().item() > 0


def test_bar_nll_fullsize_matches_oracle(cuda_device):
    """256000 query rows x 100 bars through pfn_bar_nll_fwd/bwd (the criterion's path) against the fp64 bounds of
    oracle/error_budget.py, element by element; a slice of rows also against the CPU oracle."""
    torch.manual_seed(14)
    NQ = (T - SEP) * B
    borders = torch.sort(torch.randn(NB + 1)).values
    crit = bar_distribution.FullSupportBarDistribution(borders).to(cuda_device)
    logits = torch.randn(NQ, NB, device=cuda_device, requires_grad=True)
    yq = (torch.randn(NQ, device=cuda_device) * 1.2).clamp(-6, 6)
    nll = crit(logits, yq)
    bd = crit.borders
    f = EB.bar_nll_fwd(logits.detach(), yq, bd, True)
    EB.check("bar_nll nll fullsize", nll.detach(), f["nll"], f["nll_bound"], EB.C_BAR)
    ref = O.bar_nll_ref(logits.detach()[:4096].cpu().double(), yq[:4096].cpu().double(), borders.double(), full_support=True)
    assert torch.allclose(f["nll"][:4096].cpu(), ref, rtol=1e-12, atol=1e-12)
    # the stored lse the backward reads: the same kernel called directly gives the criterion's nll bit for bit
    nll2, lse = torch.empty(NQ, device=cuda_device), torch.empty(NQ, device=cuda_device)
    idx = torch.empty(NQ, device=cuda_device, dtype=torch.int64)
    L.bar_nll_fwd(logits.detach(), yq, bd, NB, True, nll2, idx, lse, torch.zeros(1, device=cuda_device, dtype=torch.int32))
    assert torch.equal(nll2, nll.detach()) and torch.equal(idx, f["idx"])
    EB.check("bar_nll lse fullsize", lse, f["lse"], f["lse_bound"], EB.C_BAR)
    nll.mean().backward()
    exact, bound = EB.bar_nll_bwd(logits.detach(), idx, lse, torch.full((NQ,), 1.0 / NQ, device=cuda_device), EB.U32)
    EB.check("bar_nll dlogits fullsize", logits.grad, exact, bound, EB.C_BAR_GRAD)


def test_gp_sampler_fullsize_factor_is_a_cholesky(cuda_device):
    """priors.fast_gp at T=1000 (notebook hyperparameters): the factor the fused kernel leaves behind satisfies L L^T = K
    and y = L z element by element, within the fp64 bounds of oracle/error_budget.py."""
    torch.manual_seed(15)
    nb = 4
    x = torch.rand(nb, T, F, device=cuda_device); z = torch.randn(nb, T, device=cuda_device)
    ls = torch.full((nb, F), .6, device=cuda_device); os_ = torch.ones(nb, device=cuda_device); nz = torch.full((nb,), 1e-4, device=cuda_device)
    y, Lf = priors.fast_gp.sample_gp(x, z, ls, os_, nz, return_factor=True)
    assert torch.isfinite(y).all() and torch.isfinite(Lf).all()
    # the draw went through without jitter: a direct launch at jitter 0 gives it bit for bit with every pivot passing
    y0, work0, info0 = torch.empty_like(y), torch.empty(nb, T, (T + 3) // 4 * 4, device=cuda_device), torch.full((nb,), -1, device=cuda_device, dtype=torch.int32)
    L.gp_sample(x, z, ls, os_, nz, 0.0, L.KERNEL_RBF, y0, work0, info0)
    assert (info0 == 0).all() and torch.equal(y0, y) and torch.equal(EB.gp_factor(work0, T), Lf)
    assert (torch.triu(Lf, 1) == 0).all() and (torch.diagonal(Lf, dim1=1, dim2=2) > 0).all()
    K, E_K = EB.gp_kernel(x, ls, os_, nz, 0.0, L.KERNEL_RBF)
    LLt, bound = EB.gp_factor_residual(Lf, E_K)
    EB.check("gp factor fullsize", LLt, K, bound, EB.C_GP_FACTOR)
    ye, yb = EB.gp_draw(Lf, z)
    EB.check("gp y fullsize", y, ye, yb, EB.C_GP_Y)
    Kr = O.gp_kernel_ref(x[:1].cpu().double(), ls[:1].cpu().double(), os_[:1].cpu().double(), nz[:1].cpu().double())
    assert torch.allclose(K[:1].cpu(), Kr, rtol=1e-12, atol=1e-15)
