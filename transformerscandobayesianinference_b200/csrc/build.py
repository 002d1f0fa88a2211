"""In-tree build of libpfn_b200.so (sm_90a only) with plain nvcc; no JIT cache, no torch extension machinery.

`python -m transformerscandobayesianinference_b200.csrc.build` or `__graft_entry__.build()`.
The shared object lands next to the package (`transformerscandobayesianinference_b200/libpfn_b200.so`) so it
travels with the repo snapshot to the GPU box.
"""
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
ROOT = os.path.dirname(PKG)
OBJ_DIR = os.path.join(HERE, "_obj")
LIB_PATH = os.path.join(PKG, "libpfn_b200.so")

SOURCES = [
    "runtime.cu",
    "optimizer.cu",
    "gemm_tc.cu",
    "gemm_simt.cu",
    "rowwise.cu",
    "bar_nll.cu",
    "attention_simt.cu",
    "attention_tc.cu",
    "attention_bwd_tc.cu",
    "gp_sampler.cu",
    "gp_fit.cu",
    "gp_mcmc.cu",
    "dropout.cu",
    "stroke_prior.cu",
    "omniglot_prior.cu",
    "bnn_prior.cu",
    "bnn_mcmc.cu",
    "knn_cv.cu",
]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]

# per-source additions: the NUTS samplers' arithmetic must be the plain IEEE sequence their CPU restatement performs
EXTRA_FLAGS = {"gp_mcmc.cu": ["-fmad=false"], "bnn_mcmc.cu": ["-fmad=false"]}


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def _headers():
    hs = [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(ROOT, "include", "pfn_b200.h"))
    return hs


def _stale(src, obj, headers):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    return any(os.path.getmtime(p) > t for p in [src] + headers)


def _compile(nvcc, src, obj, log_dir):
    cmd = [nvcc] + NVCC_FLAGS + EXTRA_FLAGS.get(os.path.basename(src), []) + ["-c", src, "-o", obj]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    with open(os.path.join(log_dir, os.path.basename(src) + ".ptxas.log"), "w") as fh:
        fh.write(" ".join(cmd) + "\n" + proc.stdout + proc.stderr)
    if proc.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{proc.stdout}\n{proc.stderr}")
    return src


def build(force=False, verbose=True):
    nvcc = _nvcc()
    os.makedirs(OBJ_DIR, exist_ok=True)
    headers = _headers()
    srcs = [os.path.join(HERE, s) for s in SOURCES if os.path.exists(os.path.join(HERE, s))]
    objs = [os.path.join(OBJ_DIR, os.path.basename(s)[:-3] + ".o") for s in srcs]
    todo = [(s, o) for s, o in zip(srcs, objs) if force or _stale(s, o, headers)]
    if todo:
        with ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
            for done in ex.map(lambda so: _compile(nvcc, so[0], so[1], OBJ_DIR), todo):
                if verbose:
                    print(f"[pfn_b200.build] compiled {os.path.basename(done)}", flush=True)
    need_link = bool(todo) or not os.path.exists(LIB_PATH) or any(
        os.path.getmtime(o) > os.path.getmtime(LIB_PATH) for o in objs)
    if need_link:
        cmd = [nvcc, "-shared", "-o", LIB_PATH] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        proc = subprocess.run(cmd, capture_output=True, text=True)
        if proc.returncode != 0:
            raise RuntimeError(f"link failed:\n{proc.stdout}\n{proc.stderr}")
        if verbose:
            print(f"[pfn_b200.build] linked {LIB_PATH}", flush=True)
    return LIB_PATH


if __name__ == "__main__":
    build(force="--force" in sys.argv)
