"""The tabular evaluation's device paths held element by element.

The PFN path runs the training kernels in a way the training tests never do: inference only (no_grad, eval mode), one
query row per context (T = p + 1, sep = p), thousands of contexts, a decoder whose logits GEMM has N = 1.  Its forward is
recorded (oracle/engine_stages.Recorder) and every stage held to its kernel's per-element fp64 bound
(StageCheck.forward), at the golden PFNs' shapes for every edge of the eval position, and at the checkpoint
architecture at the notebook's batch.  A context's output must not depend on which other contexts share its forward:
chunked forwards and the largest single forward (about 2^20 tokens) must give every context the bits of a small batch.

The KNN kernel (csrc/knn_cv.cu) is compared bit for bit with the fp64 restatement tabular_oracle.knn_grid_search at
training-row and test-row counts that make its 256-thread loops take a second pass, on exact distance ties, with
problems that are not OK sharing the launch.  (The kernel's FEW_MEMBERS status is unreachable with labels 0 / 1:
n_splits = min(5, n // 2) and the two class counts sum to n >= 2 n_splits, so one class always has n_splits members.)"""
import os

import numpy as np
import pytest
import torch

from transformerscandobayesianinference_b200 import _lib as L, encoders, engine, tabular
from transformerscandobayesianinference_b200.transformer import TransformerModel
from oracle import engine_stages as ES, tabular_oracle as TO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = torch.load(os.path.join(ROOT, "tests", "golden", "tabular.pt"), weights_only=False)
BPTT, NS, MF = GOLDEN["bptt"], GOLDEN["max_samples"], GOLDEN["max_features"]
POSITIONS = [1, 2, 10, 30, 64, 99]
# the checkpoint architecture (the notebook's models): E 512, 4 heads of 128, nhid 1024, 5 layers, 60 features
CKPT = {"E": 512, "H": 4, "nhid": 1024, "L": 5, "F": 60}


@pytest.fixture(autouse=True)
def _on_cuda(cuda_device):
    """Every test here runs the kernels on cuda:0."""


def _golden_model(key, precision):
    c = GOLDEN["pfn"][key]["case"]
    m = TransformerModel(encoders.Linear(MF, c["E"]), 1, c["E"], c["H"], c["nhid"], c["L"], 0.0,
                         y_encoder=encoders.Linear(1, c["E"]))
    m.load_state_dict(TO.seeded_state_dict(m, c["seed"]))
    m.precision = precision
    return m.cuda()


def _ckpt_model(precision, seed=7):
    """The checkpoint architecture with seeded_state_dict weights: linear2 and out_proj are nonzero."""
    m = TransformerModel(encoders.Linear(CKPT["F"], CKPT["E"]), 1, CKPT["E"], CKPT["H"], CKPT["nhid"], CKPT["L"], 0.0,
                         y_encoder=encoders.Linear(1, CKPT["E"]))
    m.load_state_dict(TO.seeded_state_dict(m, seed))
    m.precision = precision
    return m.cuda()


def _dataset():
    name, X, y, cat = GOLDEN["datasets"][0]
    return torch.cat([X, torch.zeros(X.shape[0], MF - X.shape[1])], -1), y, cat, X.shape[1] / MF


def _checked_position(model, X, y, p, rescale, S, precision, tag):
    """tabular.evaluate_position recorded; every stage of its one forward checked.  Returns the checker.  The per-sample
    AUC is not computed: near p = bptt a sample's few test rows can hold one class, where the AUC is undefined."""
    rec = ES.Recorder(L).install()
    try:
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(tabular, "metric_used", lambda y, s: np.zeros(np.shape(y)[:-1]))
            _, outputs, _ = tabular.evaluate_position(X, y, [], model, BPTT, p, rescale_features=rescale, max_samples=S)
    finally:
        rec.remove()
    torch.cuda.synchronize()
    calls = rec.calls
    eval_xs, eval_ys = TO.windows(X, y, BPTT, S)
    Q = BPTT - p
    xs, ys = tabular.pfn_contexts(eval_xs.cuda(), eval_ys.cuda(), p, rescale)
    # the embedding reads the contexts of pfn_contexts bit for bit: column q * S + s is sample s with its test row p + q
    a = calls[0].a
    assert calls[0].fn == "embed_fwd" and (a["T"], a["B"], a["sep"]) == (p + 1, Q * S, p)
    assert torch.equal(a["x"], xs) and torch.equal(a["y"], ys)
    assert torch.equal(a["y"][:p].reshape(p, Q, S), eval_ys[:p].cuda().float().unsqueeze(1).expand(p, Q, S))
    ref, _ = TO.pfn_contexts_ref(eval_xs, eval_ys, p, rescale)          # the layout, against the oracle's
    assert torch.allclose(a["x"].cpu().double(), ref, rtol=2 ** -23, atol=1e-6)
    layers = [dict(zip(ES.LAYER_PARAM_NAMES, [t.detach() for t in engine.layer_params(l)]))
              for l in model.transformer_encoder.layers]
    paths = {"u_is_grad": precision == "bf16" and engine._GELU_GRAD_FWD, "rowdot": False, "fused_bias": False}
    chk = ES.StageCheck(T=p + 1, B=Q * S, H=model.nhead, sep=p, thr=0, mask=None, num_sms=L.num_sms(), paths=paths,
                        tag=f"{tag}: ")
    logits = chk.forward(calls, x=xs, y=ys, precision=precision, layers=layers,
                         emb=(model.encoder.weight.detach(), model.encoder.bias.detach(),
                              model.y_encoder.weight.detach(), model.y_encoder.bias.detach()),
                         dec=(model.decoder[0].weight.detach(), model.decoder[0].bias.detach(),
                              model.decoder[2].weight.detach(), model.decoder[2].bias.detach()))
    # the outputs are the sigmoid of the recorded logits, bit for bit
    want = torch.sigmoid(logits[:, 0]).reshape(Q, S).double().cpu().numpy()
    np.testing.assert_array_equal(outputs, want)
    return chk


# ---------------------------------------------------------------------------------------------------------------------
# (a) the golden PFNs at every edge of the eval position
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", ["dh128", "dh64"])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_tabular_forward_stages_golden_models(capsys, key, precision):
    """dh128: one head of 128 (tensor-core attention in bf16); dh64: two heads of 64 (SIMT attention)."""
    model = _golden_model(key, precision)
    X, y, _, rescale = _dataset()
    worst = {}
    for p in POSITIONS:
        chk = _checked_position(model, X, y, p, rescale, NS, precision, f"{key} {precision} p={p}")
        for stage, r in chk.worst.items():
            worst[stage] = max(worst.get(stage, 0.0), r)
    with capsys.disabled():
        print()
        for stage, r in worst.items():
            print(f"[tabular-stages] {key} {precision} p={POSITIONS}: {stage}: worst err/bound = {r:.4g}")


# ---------------------------------------------------------------------------------------------------------------------
# (b) the checkpoint architecture at the notebook's batch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("p", [30, 99])
def test_tabular_forward_stages_checkpoint_shape(capsys, precision, p):
    """bptt 100, 20 samples: p = 30 is 1 400 contexts of 31 tokens, p = 99 is 20 contexts of 100 tokens.  The fp64 work
    of the checks runs on the device."""
    model = _ckpt_model(precision)
    g = torch.Generator().manual_seed(11)
    S = 20
    X = torch.randn(BPTT + S, CKPT["F"], generator=g)
    y = (torch.rand(BPTT + S, generator=g) < 0.5).float()
    chk = _checked_position(model, X, y, p, 1.0, S, precision, f"ckpt {precision} p={p}")
    with capsys.disabled():
        print()
        chk.report(f"[tabular] ckpt {precision} p={p} ({(BPTT - p) * S} contexts of {p + 1} tokens)")


# ---------------------------------------------------------------------------------------------------------------------
# (c) batch independence: chunked forwards, and the largest single forward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", ["dh128", "dh64"])
def test_tabular_chunked_forwards_equal_one_forward(monkeypatch, key):
    """MAX_FORWARD_TOKENS set for chunks of 600 contexts (the last one 200) and for one context per chunk: every output
    equals the one-forward output bit for bit."""
    model = _golden_model(key, "bf16")
    X, y, cat, rescale = _dataset()
    p = 30
    run = lambda: tabular.evaluate_position(X, y, cat, model, BPTT, p, rescale_features=rescale, max_samples=NS)[1]
    one = run()
    assert one.shape == (BPTT - p, NS)
    for per in (600, 1):
        monkeypatch.setattr(tabular, "MAX_FORWARD_TOKENS", per * (p + 1))
        L.reset_launch_count()
        chunked = run()
        launches = L.launch_count()
        np.testing.assert_array_equal(chunked, one)
        monkeypatch.undo()
        L.reset_launch_count()
        run()
        assert launches == -(-(BPTT - p) * NS // per) * L.launch_count()      # one forward per chunk


def test_tabular_largest_forward_is_batch_independent(capsys):
    """The checkpoint architecture in bf16 at the largest forward _pfn_outputs runs: 70 test rows x 483 samples =
    33 810 contexts of 31 tokens, 1 048 110 tokens (qkv holds 1.61e9 elements).  72 contexts spread over the batch, the
    first and the last included, run again as a batch of their own must give the same bits."""
    model = _ckpt_model("bf16")
    p, T, S = 30, 100, 483
    Q = T - p
    assert Q * S * (p + 1) <= tabular.MAX_FORWARD_TOKENS < Q * (S + 1) * (p + 1)      # one more sample: two forwards
    g = torch.Generator().manual_seed(12)
    eval_xs = torch.randn(T, S, CKPT["F"], generator=g).cuda()
    eval_ys = (torch.rand(T, S, generator=g) < 0.5).float().cuda()
    L.reset_launch_count()
    big = tabular._pfn_outputs(model, eval_xs, eval_ys, p, 1.0).reshape(-1)      # context q * S + s
    one_forward = L.launch_count()
    idx = torch.unique(torch.cat([torch.linspace(0, Q * S - 1, 64).round().long(),
                                  torch.randint(0, Q * S, (8,), generator=g), torch.tensor([1, Q * S - 2])]))
    xs, ys = tabular.pfn_contexts(eval_xs, eval_ys, p)
    sel = idx.cuda()
    with torch.no_grad():
        L.reset_launch_count()
        logits = model((xs[:, sel].contiguous(), ys[:, sel].contiguous()), single_eval_pos=p)
        assert L.launch_count() == one_forward                                   # the big batch was one forward
    small = torch.sigmoid(logits.float()).reshape(-1).double().cpu().numpy()
    differ = np.flatnonzero(small != big[idx.numpy()])
    with capsys.disabled():
        print(f"\n[tabular] largest forward: {Q * S} contexts, {Q * S * (p + 1)} tokens; {len(idx)} contexts compared, "
              f"{len(differ)} differ from a batch of {len(idx)}")
    assert len(differ) == 0, f"contexts {idx[differ].tolist()} differ: {big[idx.numpy()][differ]} vs {small[differ]}"


# ---------------------------------------------------------------------------------------------------------------------
# (d) the KNN kernel against the fp64 grid search, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
# (n training rows, m test rows, F features): n = 5 and 7 have a CV candidate k larger than a fold's training set;
# 255 / 256 / 257 and 1024 rows or test rows make the CTA's 256 threads take one, one or two, and four passes
KNN_SIZES = [(4, 1, 1), (5, 255, 60), (6, 256, 1), (7, 257, 60), (11, 1, 1024), (255, 257, 1), (256, 1, 60),
             (257, 256, 1024), (1024, 257, 60), (1024, 255, 1)]
# problem kinds of one launch: OK ones, then two the kernel must refuse
OK_KINDS = ["random", "row0_is_1", "singleton_class", "integer_ties", "duplicated_rows"]
BAD_KINDS = {"bad_label": L.KNN_BAD_LABEL, "one_class": L.KNN_ONE_CLASS}


def _knn_problem(kind, n, m, F, g):
    x = torch.randn(n + m, F, generator=g)
    y = (torch.rand(n, generator=g) < 0.5).float()
    y[:2] = torch.tensor([0.0, 1.0])
    y = y[torch.randperm(n, generator=g)]
    if kind == "row0_is_1":
        y[0] = 1.0
        if bool((y == 1).all()):
            y[1] = 0.0
    elif kind == "singleton_class":
        y = torch.zeros(n)
        y[int(torch.randint(0, n, (1,), generator=g))] = 1.0
    elif kind == "integer_ties":
        x = torch.randint(0, 3, (n + m, F), generator=g).float()
    elif kind == "duplicated_rows":
        x = torch.randint(-2, 3, (n + m, F), generator=g).float()
        src = torch.randint(0, n, (n + m,), generator=g)
        dup = torch.rand(n + m, generator=g) < 0.5
        x[dup] = x[src[dup]]
    elif kind == "bad_label":
        y[n // 2] = 0.5
    elif kind == "one_class":
        y = torch.ones(n)
    return x, y


def _knn_launch(x, y):
    rows, S, F = x.shape
    n = y.shape[0]
    m, K = rows - n, min(L.KNN_MAX_K, n - 2)
    out = (torch.full((m, S), -1.0, dtype=torch.float64, device="cuda"), torch.full((S,), -1, dtype=torch.int32, device="cuda"),
           torch.full((S, K), -1.0, dtype=torch.float64, device="cuda"), torch.full((S,), -1, dtype=torch.int32, device="cuda"))
    L.knn_cv(x.cuda().contiguous(), y.cuda().contiguous(), *out)
    return [t.cpu() for t in out]


@pytest.mark.parametrize("n,m,F", KNN_SIZES)
def test_knn_kernel_matches_the_grid_search_bitwise(n, m, F):
    g = torch.Generator().manual_seed(n * 7919 + m * 31 + F)
    kinds = OK_KINDS + list(BAD_KINDS)
    probs = [_knn_problem(k, n, m, F, g) for k in kinds]
    x = torch.stack([p[0] for p in probs], 1)
    y = torch.stack([p[1] for p in probs], 1)
    proba, k_best, cv_mean, status = _knn_launch(x, y)
    nok = len(OK_KINDS)
    nan_candidates = 0
    for s, kind in enumerate(kinds):
        if kind in BAD_KINDS:
            assert int(status[s]) == BAD_KINDS[kind], (kind, int(status[s]))
            assert int(k_best[s]) == 0 and bool(proba[:, s].isnan().all()) and bool(cv_mean[s].isnan().all()), kind
            continue
        assert int(status[s]) == L.KNN_OK, (kind, int(status[s]))
        r_proba, r_k, r_mean, _ = TO.knn_grid_search(x[:n, s].numpy(), y[:, s].numpy(), x[n:, s].numpy())
        assert int(k_best[s]) == r_k, (kind, int(k_best[s]), r_k)
        np.testing.assert_array_equal(cv_mean[s].numpy(), r_mean, err_msg=kind)           # NaN where NaN
        np.testing.assert_array_equal(proba[:, s].numpy(), r_proba, err_msg=kind)
        nan_candidates += int(np.isnan(r_mean).sum())
    assert (nan_candidates > 0) == (n in (5, 7))
    # the refused problems leave their neighbours' results alone: the OK problems alone give the same bits
    bits = lambda t: t.contiguous().view(torch.int64) if t.dtype == torch.float64 else t
    alone = _knn_launch(x[:, :nok].clone(), y[:, :nok].clone())
    for got, ref in zip(alone, (proba[:, :nok], k_best[:nok], cv_mean[:nok], status[:nok])):
        assert torch.equal(bits(got), bits(ref))
