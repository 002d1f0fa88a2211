"""The persistent wgmma GEMM at the activation GEMMs' short contractions (K = 512 / 1024 / 1536, no split-K): every
epilogue kind, ragged M and N edges, unit counts that are not a multiple of the grid, CTAs that run one unit and CTAs
that run several.  Each output is held to the per-element fp64 bounds of oracle/error_budget.py and, because a tile's
k-blocks are summed in a fixed order, to the exact bytes recorded in tests/golden/gemm_short_k.json
(tools/make_gemm_short_k_golden.py holds the cases and makes that file)."""
import json
import os
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_gemm_short_k_golden as G
from transformerscandobayesianinference_b200 import _lib as L
from oracle import error_budget as EB


@pytest.mark.parametrize("name", sorted(G.CASES))
def test_gemm_short_k(name, cuda_device):
    M, N, K, epi, b_mn, c2, has_bias, has_aux, f32 = G.CASES[name]
    (A, B, bias, aux), out = G.run(name, L)
    C = out["C"]
    u = EB.U32 if f32 else EB.U
    if epi == "rowdot":
        ref, bound, _ = EB.gemm(A, B, u, EB.C_ACC_TC)
        EB.check(f"{name} C", C, ref, bound, EB.C_GEMM)
        exact, bound = EB.rowdot(C, aux, G.ROWDOT_WIDTH)
        EB.check(f"{name} rowdot", out["rowdot"], exact, bound, EB.C_ROWDOT)
    else:
        ref, bound, _ = EB.gemm(A, B, u, EB.C_ACC_TC, bias=bias, aux=aux, epilogue=epi)
        EB.check(f"{name} C", C, ref, bound, EB.C_GEMM)
    if c2 == "grad":
        ref, bound, _ = EB.gemm(A, B, EB.U, EB.C_ACC_TC, bias=bias, epilogue="gelu_grad")
        EB.check(f"{name} C2", out["C2"], ref, bound, EB.C_GEMM)
    elif c2 == "pre":
        ref, bound, _ = EB.gemm(A, B, EB.U, EB.C_ACC_TC, bias=bias)
        EB.check(f"{name} C2", out["C2"], ref, bound, EB.C_GEMM)

    with open(G.GOLDEN) as fh:
        golden = json.load(fh)[name]
    assert sorted(golden) == sorted(out)
    for k, t in out.items():
        assert G.digest(t) == golden[k], f"{name}: {k} differs from the recorded bytes"
