"""Cases of tests/test_gpu_gemm_short_k.py and the maker of their golden hashes (tests/golden/gemm_short_k.json).

The cases are the persistent wgmma GEMM at the short contractions of the activation GEMMs (K = 512 / 1024 / 1536, one
unit per 128 x 128 tile, no split-K) with every epilogue kind, ragged M and N edges, and unit counts that leave one unit
per CTA or several (on a 132-SM H100: 408 units, not a multiple of the grid; 96 units, one per CTA).  A tile's k-blocks
are summed in the same order whatever the schedule, so every output is a fixed function of the inputs: the golden file
holds the SHA-256 of each output's bytes as a given build of the library produced them, and the test requires the same
bytes from the current build.

    python tools/make_gemm_short_k_golden.py [path/to/libpfn_b200.so]     (needs a CUDA device)"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

GOLDEN = os.path.join(ROOT, "tests", "golden", "gemm_short_k.json")

# name: (M, N, K, epilogue, B MN-major, C2 ("grad" = gelu', "pre" = pre-activation, None), bias, aux, fp32 C)
CASES = {
    "qkv_bias_k512": (4281, 1536, 512, "none", False, None, True, False, False),
    "outproj_bias_aux_k512": (4281, 512, 512, "none", False, None, True, True, False),
    "gelu_c2grad_k512": (4281, 1024, 512, "gelu", False, "grad", True, False, False),
    "gelu_c2pre_k1024_ragged_n": (1000, 328, 1024, "gelu", False, "pre", True, False, False),
    "gelu_c2grad_aux_k512": (2000, 256, 512, "gelu", False, "grad", True, True, False),
    "gelu_k1536_ragged_n": (3000, 200, 1536, "gelu", False, None, True, False, False),
    "gelu_c2grad_k1536_one_unit_per_cta": (1000, 1536, 1536, "gelu", False, "grad", True, False, False),
    "lin2_bias_aux_k1024": (4281, 512, 1024, "none", False, None, True, True, False),
    "du_dgrad_mul_k512": (4281, 1024, 512, "mul", True, None, False, True, False),
    "dh1_dgrad_aux_k1024": (4281, 512, 1024, "none", True, None, False, True, False),
    "dattn_dgrad_rowdot_k512": (4281, 512, 512, "rowdot", True, None, False, True, False),
    "dh2_dgrad_aux_k1536": (4281, 512, 1536, "none", True, None, False, True, False),
    "gelu_bwd_dgrad_k512": (2999, 1024, 512, "gelu_bwd", True, None, False, True, False),
    "f32_out_aux_k512_ragged_n": (4281, 328, 512, "none", False, None, True, True, True),
}
ROWDOT_WIDTH = 128


def inputs(name):
    """The case's operands, drawn on the host from a seed derived from its name, on the current CUDA device.  B is the
    [N, K] logical operand; for a B MN-major case it is stored as its [K, N] transpose."""
    M, N, K, epi, b_mn, c2, has_bias, has_aux, f32 = CASES[name]
    g = torch.Generator().manual_seed(int.from_bytes(hashlib.sha256(name.encode()).digest()[:4], "little"))
    dev = torch.device("cuda")
    A = torch.randn(M, K, generator=g).to(torch.bfloat16).to(dev)
    B = (torch.randn(N, K, generator=g) * K ** -0.5).to(torch.bfloat16).to(dev)
    bias = torch.randn(N, generator=g).to(dev) if has_bias else None
    aux = None
    if has_aux:
        aux = torch.randn(M, N, generator=g)
        if epi == "mul":
            aux = torch.sigmoid(aux)
        aux = aux.to(torch.bfloat16).to(dev)
    return A, B, bias, aux


def run(name, lib):
    """Run the case on the library module `lib` (transformerscandobayesianinference_b200._lib); returns (inputs, outputs)
    with outputs a dict of named result tensors."""
    M, N, K, epi, b_mn, c2, has_bias, has_aux, f32 = CASES[name]
    A, B, bias, aux = inputs(name)
    dev = A.device
    C = torch.empty(M, N, device=dev, dtype=torch.float32 if f32 else torch.bfloat16)
    out = {"C": C}
    kw = dict(bias=bias, aux=aux, use_tc=True, M=M, N=N, K=K)
    if b_mn:
        kw["b_mn_major"] = True
        Bop = B.t().contiguous()
    else:
        Bop = B
    if epi == "gelu":
        kw["epilogue"] = lib.EPI_GELU
        if c2 is not None:
            out["C2"] = kw["C2"] = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            kw["c2_gelu_grad"] = c2 == "grad"
    elif epi == "mul":
        kw["epilogue"] = lib.EPI_MUL
    elif epi == "gelu_bwd":
        kw["epilogue"] = lib.EPI_GELU_BWD
    elif epi == "rowdot":
        out["rowdot"] = torch.zeros(M, N // ROWDOT_WIDTH, device=dev)
        kw["epilogue"] = lib.EPI_ROWDOT
        kw["rowdot"] = (out["rowdot"], ROWDOT_WIDTH)
    lib.gemm(A, Bop, C, **kw)
    torch.cuda.synchronize()
    return (A, B, bias, aux), out


def digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()


def main():
    if not torch.cuda.is_available():
        raise SystemExit("make_gemm_short_k_golden.py needs a CUDA device")
    if len(sys.argv) > 1:
        os.environ["PFN_B200_LIB"] = os.path.abspath(sys.argv[1])
    from transformerscandobayesianinference_b200 import _lib as L
    golden = {name: {k: digest(v) for k, v in run(name, L)[1].items()} for name in CASES}
    with open(GOLDEN, "w") as fh:
        json.dump(golden, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print(f"wrote {len(golden)} cases to {GOLDEN}")


if __name__ == "__main__":
    main()
