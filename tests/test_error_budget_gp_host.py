"""The GP sampler bounds of oracle/error_budget.py on a float32 CPU restatement of csrc/gp_sampler.cu that rounds where
the kernel rounds (left-looking, panel width 32, the update's fmaf chain over the finished panels, K^ - acc, the warp
Cholesky of the diagonal block, the row solve through fl(1 / L_jj), one 32-term dot per panel into y): the restatement
lies inside the bounds at c = 1, and each numerical slip a kernel could make falls outside them at the constants the GPU
tests use.  Each slip also reports whether the max-scaled tolerances the GPU tests used before pass it."""
import math

import pytest
import torch

from oracle import error_budget as EB

F32 = torch.float32
NB = EB.GP_PANEL
RBF, M12, M32, M52 = EB.GP_RBF, EB.GP_MATERN12, EB.GP_MATERN32, EB.GP_MATERN52
NAMES = {RBF: "rbf", M12: "matern12", M32: "matern32", M52: "matern52"}


def _fma(a, b, c):
    """fp32 fma: the product of two fp32 values is exact in fp64, so one rounding of the fp64 sum."""
    return (a.double() * b.double() + c.double()).float()


def _exp(x, fast):
    if not fast:
        return torch.exp(x)
    t = x * torch.tensor(math.log2(math.e), dtype=F32)      # ex2.approx(x log2 e): the rounded argument
    return torch.exp2(t.double()).float()


def kernel_matrix(x, ls, os_, noise, jitter, kt, slip=None):
    """K^ [B, T, T] as gp_kernel_value and its caller form it in fp32."""
    B, T, Fd = x.shape
    il = 1.0 / ls
    if slip == "inv_ls_bf16":
        il = il.bfloat16().float()
    xs = x * il.unsqueeze(1)
    d2 = torch.zeros(B, T, T, dtype=F32)
    for f in range(Fd):
        df = xs[:, :, f].unsqueeze(2) - xs[:, :, f].unsqueeze(1)
        d2 = _fma(df, df, d2)
    o = os_.view(B, 1, 1)
    fast = slip == "fast_exp"
    if kt == RBF:
        k = o * _exp(-0.5 * d2, fast)
    else:
        r = torch.sqrt(d2)
        if kt == M12:
            k = o * _exp(-r, fast)
        elif kt == M32:
            a = torch.tensor(1.732 if slip == "matern32_1732" else 1.7320508075688772, dtype=F32) * r
            k = o * (1.0 + a) * _exp(-a, fast)
        else:
            a = torch.tensor(2.23606797749979, dtype=F32) * r
            c53 = torch.tensor(5.0 / 3.0 + (1e-5 if slip == "matern52_5_3" else 0.0), dtype=F32)
            k = o * _fma(c53, d2, 1.0 + a) * _exp(-a, fast)
    nz = noise.clone()
    if slip == "noise_dataset0":
        nz[:] = noise[0]
    j = {"jitter_dropped": 0.0, "jitter_doubled": 2.0 * jitter}.get(slip, jitter)
    diag = os_ + (nz + torch.tensor(j, dtype=F32))
    eye = torch.eye(T, dtype=torch.bool)
    return torch.where(eye, diag.view(B, 1, 1), k)


def sample(x, z, ls, os_, noise, jitter, kt, slip=None):
    """(y [B, T], L [B, T, T], info [B]) in the kernel's order of operations."""
    K = kernel_matrix(x, ls, os_, noise, jitter, kt, slip)
    B, T, _ = K.shape
    Lm = torch.zeros(B, T, T, dtype=F32)
    y = torch.zeros(B, T, dtype=F32)
    info = torch.zeros(B, dtype=torch.int64)
    lane = torch.arange(NB)
    for c0 in range(0, T, NB):
        nb = min(NB, T - c0)
        acc = torch.zeros(B, T - c0, nb, dtype=F32)
        for k in range(c0):
            if slip == "drop_last_chunk" and k >= c0 - NB:
                break
            acc = _fma(Lm[:, c0:, k].unsqueeze(2), Lm[:, c0:c0 + nb, k].unsqueeze(1), acc)
        U = K[:, c0:, c0:c0 + nb] - acc
        # diagonal block: one warp, lane = row, unit rows past the matrix edge
        row = torch.zeros(B, NB, NB, dtype=F32)
        row[:, :nb, :nb] = U[:, :nb]
        row[:, lane >= nb] = torch.eye(NB, dtype=F32)[lane >= nb]
        for j in range(NB):
            djj = row[:, j, j]
            bad = ~(djj > 0)
            info = torch.where(bad & (info == 0), torch.full_like(info, c0 + j + 1), info)
            ljj = torch.sqrt(torch.where(bad, torch.ones_like(djj), djj))
            lij = torch.where(lane > j, row[:, :, j] / ljj.unsqueeze(1),
                              torch.where(lane == j, ljj.unsqueeze(1).expand(B, NB), torch.zeros(B, NB)))
            row[:, :, j] = lij
            if j + 1 < NB:
                upd = _fma(-lij.unsqueeze(2), lij[:, j + 1:].unsqueeze(1), row[:, :, j + 1:])
                row[:, :, j + 1:] = torch.where(lane.view(NB, 1) >= lane[j + 1:].view(1, -1), upd, row[:, :, j + 1:])
        sL = torch.tril(row)
        sLinv = 1.0 / torch.diagonal(sL, dim1=1, dim2=2)
        Lm[:, c0:c0 + nb, c0:c0 + nb] = sL[:, :nb, :nb]
        if T > c0 + NB:
            R = U[:, NB:]
            v = torch.zeros_like(R)
            for c in range(NB):
                a = R[:, :, c]
                for p in range(c):
                    a = _fma(-v[:, :, p], sL[:, c, p].unsqueeze(1), a)
                v[:, :, c] = a * sLinv[:, c].unsqueeze(1)
            Lm[:, c0 + NB:, c0:c0 + NB] = v
        if slip == "drop_last_partial_y" and nb < NB:
            continue
        dot = torch.zeros(B, T - c0, dtype=F32)
        for c in range(nb):
            dot = _fma(Lm[:, c0:, c0 + c], z[:, c0 + c].unsqueeze(1), dot)
        y[:, c0:] = y[:, c0:] + dot
    return y, Lm, info


def _data(B, T, Fd, seed, spans=True):
    """Per-dataset hyperparameters log-uniform over outputscale 1e-6..50, noise 1e-4..50, lengthscale 0.02..5 (spans), or
    the moderate ones of the LAPACK comparisons."""
    g = torch.Generator().manual_seed(seed)
    lu = lambda lo, hi, *s: torch.exp(math.log(lo) + (math.log(hi) - math.log(lo)) * torch.rand(*s, generator=g, dtype=torch.float64)).float()
    x = torch.rand(B, T, Fd, generator=g)
    z = torch.randn(B, T, generator=g)
    if spans:
        ls, os_, noise = lu(0.02, 5.0, B, Fd), lu(1e-6, 50.0, B), lu(1e-4, 50.0, B)
    else:
        ls = (torch.rand(B, Fd, generator=g) * 0.5 + 0.1)
        os_, noise = torch.rand(B, generator=g) + 0.5, torch.rand(B, generator=g) * 0.2 + 0.05
    return x, z, ls, os_, noise


def _check_all(x, z, ls, os_, noise, jitter, kt, y, Lm, info, c_f, c_y, tag, verbose=True):
    """Factor and draw ratios (factor only where every pivot passed)."""
    K, E_K = EB.gp_kernel(x, ls, os_, noise, jitter, kt)
    ok = info == 0
    rf = 0.0
    if ok.any():
        assert (torch.diagonal(Lm[ok], dim1=1, dim2=2) > 0).all()
        LLt, bound = EB.gp_factor_residual(Lm[ok], E_K[ok])
        rf = EB.check(f"host gp factor {tag}", LLt, K[ok], bound, c_f, verbose)
    ye, yb = EB.gp_draw(Lm, z)
    ry = EB.check(f"host gp y {tag}", y, ye, yb, c_y, verbose)
    return rf, ry


CASES = [(1, 1, RBF, 0.0), (2, 3, M12, 1e-6), (5, 18, M32, 1e-4), (31, 128, M52, 0.05), (33, 1, RBF, 1e-4), (64, 3, M52, 0.0),
         (65, 1, M32, 0.05), (97, 18, M12, 0.0), (130, 1, M52, 1e-6), (130, 3, RBF, 0.05)]


@pytest.mark.parametrize("T,Fd,kt,jitter", CASES, ids=[f"T{c[0]}-F{c[1]}-{NAMES[c[2]]}-j{c[3]:g}" for c in CASES])
def test_gp_restatement_inside_bound_at_c1(T, Fd, kt, jitter):
    x, z, ls, os_, noise = _data(6, T, Fd, T + Fd)
    y, Lm, info = sample(x, z, ls, os_, noise, jitter, kt)
    assert (info == 0).sum() >= 3, info
    _check_all(x, z, ls, os_, noise, jitter, kt, y, Lm, info, 1.0, 1.0, f"T={T} F={Fd} {NAMES[kt]}")


def test_gp_restatement_bound_has_underflow_floor():
    """ls = 0.05 on [0, 1): most pairs' kernel values underflow in fp32 but not in fp64; the bound's absolute floor holds them."""
    x, z, _, _, noise = _data(3, 100, 1, 7)
    ls = torch.full((3, 1), 0.05)
    os_ = torch.tensor([1e-6, 1.0, 50.0])
    for kt in (RBF, M12, M32, M52):
        y, Lm, info = sample(x, z, ls, os_, noise, 0.0, kt)
        _check_all(x, z, ls, os_, noise, 0.0, kt, y, Lm, info, 1.0, 1.0, f"ls=0.05 {NAMES[kt]}")


def test_gp_restatement_info_is_first_failing_pivot():
    """Points 150 apart (every off-diagonal kernel value is 0 in fp32), duplicated rows give exact zero pivots."""
    T = 130
    x = (150.0 * torch.arange(T, dtype=F32)).view(1, T, 1).repeat(4, 1, 1)
    for b, ks in enumerate(((1,), (32, 65), (128, 33), (T - 1,))):
        for k in ks:
            x[b, k] = x[b, k - 1]
    ones = torch.ones(4)
    for kt in (RBF, M12, M32, M52):
        _, _, info = sample(x, torch.randn(4, T), torch.ones(4, 1), ones, torch.zeros(4), 0.0, kt)
        assert info.tolist() == [2, 33, 34, T]


# name, (T, F, kernel, jitter, data), slip.  "dyadic": x on a 1/64 grid and lengthscale 1/8, so that d2 is exact in fp32
# and the bound holds only expf's and the constants' errors
SLIPS = [
    ("matern32_1732", (65, 1, M32, 0.0, "moderate")),
    ("matern52_5_3", (65, 1, M52, 0.0, "dyadic")),
    ("noise_dataset0", (65, 3, RBF, 0.0, "spans")),
    ("jitter_dropped", (65, 1, M52, 0.05, "moderate")),
    ("jitter_doubled", (65, 1, M52, 0.05, "moderate")),
    ("fast_exp", (65, 1, RBF, 0.0, "dyadic")),
    ("inv_ls_bf16", (65, 3, M32, 0.0, "moderate")),
    ("drop_last_chunk", (130, 1, M12, 0.0, "moderate")),
    ("drop_last_partial_y", (130, 1, RBF, 0.0, "moderate")),
]


def _slip_data(T, Fd, kind):
    x, z, ls, os_, noise = _data(6, T, Fd, 11, kind == "spans")
    if kind == "dyadic":
        g = torch.Generator().manual_seed(12)
        x = torch.randint(0, 64, (6, T, Fd), generator=g).float() / 64
        ls = torch.full_like(ls, 0.125)
    return x, z, ls, os_, noise


@pytest.mark.parametrize("name,case", SLIPS, ids=[s[0] for s in SLIPS])
def test_gp_slip_outside_bound(name, case):
    T, Fd, kt, jitter, kind = case
    x, z, ls, os_, noise = _slip_data(T, Fd, kind)
    _, _, info_ok = sample(x, z, ls, os_, noise, jitter, kt)
    assert (info_ok == 0).all()
    y, Lm, info = sample(x, z, ls, os_, noise, jitter, kt, slip=name)
    ok = info == 0
    K, E_K = EB.gp_kernel(x, ls, os_, noise, jitter, kt)
    LLt, bound = EB.gp_factor_residual(Lm[ok], E_K[ok])
    # a pivot that fails only under the slip is caught by the info check
    rf = math.inf if not ok.all() else (LLt - K[ok]).abs().div(bound).max().item()
    ye, yb = EB.gp_draw(Lm, z)
    ry = (y.double() - ye).abs().div(yb).max().item()
    # the old checks: max |L L^T - K| <= 2e-5 max |K| over the batch, |y - y_LAPACK| <= 5e-3 max |y_LAPACK|
    old_f = ok.all().item() and (LLt - K[ok]).abs().max().item() <= 2e-5 * K.abs().max().item()
    yr = (torch.linalg.cholesky(K) @ z.double().unsqueeze(-1)).squeeze(-1)
    old_y = (y.double() - yr).abs().max().item() <= 5e-3 * yr.abs().max().item()
    print(f"[perturbation] gp {name}: factor err/bound {rf:.3g} (c {EB.C_GP_FACTOR}), y err/bound {ry:.3g} "
          f"(c {EB.C_GP_Y}); old tolerances {'PASS' if old_f and old_y else 'fail'} (factor {old_f}, y {old_y})")
    assert rf > EB.C_GP_FACTOR or ry > EB.C_GP_Y
