"""The input-gradient binding (_lib_input_grad.py) against its header (include/pfn_b200_input_grad.h), on the host.

Without the built library: the ctypes descriptor has the size and member offsets of its header struct as the host C
compiler lays it out, `_PROTOTYPES` has every prototype's parameter kinds, and every wrapper's calls match the log in
tests/golden/lib_calls_input_grad.json (entry points in order, arguments and descriptors field by field with pointers
as the name of the argument tensor they point into, launches counted, tensors checked), recorded against a fake of the
library (`python tests/test_input_grad_cabi_host.py` rewrites it).  A CPU tensor in any argument is rejected before the
library is called.  With the built library: it exports every entry point the header declares."""
import ctypes
import inspect
import json
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from transformerscandobayesianinference_b200 import _lib as L, _lib_input_grad as LIG  # noqa: E402

HEADER = os.path.join(ROOT, "include", "pfn_b200_input_grad.h")
GOLDEN = os.path.join(ROOT, "tests", "golden", "lib_calls_input_grad.json")
BF16, F32, I32 = torch.bfloat16, torch.float32, torch.int32
STREAM = object()
C_TYPES = {"int": ctypes.c_int, "float": ctypes.c_float}


def t(*shape, dtype=F32):
    return torch.zeros(shape, dtype=dtype)


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def _ctype(decl):
    return " ".join(decl.replace("*", " * ").split()[:-1]).replace(" *", "*")


def _prototypes():
    out = {}
    for chunk in _header().split(";"):
        m = re.fullmatch(r"\s*([^{}()#]*?)\s*\b(pfn_\w+)\s*\(([^()]*)\)\s*", chunk)
        if m:
            out[m.group(2)] = [p for p in m.group(3).split(",") if p.strip() != "void"]
    return out


def test_struct_layout_matches_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler (cc / gcc)")
    tags = re.findall(r"typedef\s+struct\s+(pfn_\w+)\s*\{", _header())
    assert tags == ["pfn_attn_ctx_grad_desc"]
    cls = LIG.AttnCtxGradDesc
    lines = [f'printf("sizeof %zu\\n", sizeof(pfn_attn_ctx_grad_desc));']
    lines += [f'printf("{n} %zu\\n", offsetof(pfn_attn_ctx_grad_desc, {n}));' for n, _ in cls._fields_]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "pfn_b200_input_grad.h"\n\nint main(void) {\n'
                   + "".join(f"  {s}\n" for s in lines) + "  return 0;\n}\n")
    r = subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    body = re.search(r"struct\s+pfn_attn_ctx_grad_desc\s*\{(.*?)\}", _header(), flags=re.S).group(1)
    names = [n.split()[-1].lstrip("*") for d in filter(str.strip, body.split(";")) for n in d.split(",")]
    assert names == [n for n, _ in cls._fields_]
    assert cls._fields_[0][1] is L.AttnCtxDesc
    assert [c for _, c in cls._fields_[1:]] == [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_void_p] * 2
    for name, _ in cls._fields_:
        assert getattr(cls, name).offset == int(out[name]), name
    assert ctypes.sizeof(cls) == int(out["sizeof"])


def test_prototypes_match_header():
    protos = _prototypes()
    assert list(LIG._PROTOTYPES) == list(protos) and len(protos) == 5
    for name, params in protos.items():
        want = []
        for p in params:
            ct = _ctype(p)
            if ct == "const pfn_attn_ctx_grad_desc*":
                want.append(ctypes.POINTER(LIG.AttnCtxGradDesc))
            else:
                want.append(ctypes.c_void_p if ct.endswith("*") else C_TYPES[ct])
        assert LIG._PROTOTYPES[name] == want, name


def test_declare_checks_every_symbol():
    class Fake:
        pass
    lib = Fake()
    for name in LIG._PROTOTYPES:
        setattr(lib, name, Fake())
    assert LIG.declare(lib) is lib
    assert lib.pfn_embed_input_bwd.restype is ctypes.c_int
    del lib.pfn_attention_ctx_bwd_tc
    with pytest.raises(RuntimeError, match="does not export pfn_attention_ctx_bwd_tc"):
        LIG.declare(lib)


def test_header_symbols_are_exported():
    lib = L.load()
    for name in LIG.EXPORTED_SYMBOLS:
        assert hasattr(lib, name), f"{name} declared in include/pfn_b200_input_grad.h but not exported"


# ---- the wrappers against a recording fake of the library ----------------------------------------------------------
def _attn(dtype, bwd, n=6, ragged=False):
    m, B, H, dh = 8, 2, 2, 4
    kv = t(n * B, 2 * H * dh, dtype=dtype) if n > 0 else None      # the cache is not read when n == 0
    a = [t(m * B, 3 * H * dh, dtype=dtype), kv, t(m * B, H * dh, dtype=dtype), t(B * H, m)]
    if bwd:
        a += [t(m * B, H * dh, dtype=dtype), t(m * B, 3 * H * dh, dtype=dtype), t(B * H, m)]
    return a + [m, n, B, H, dh, t(B, dtype=I32) if ragged else None]


CASES = [
    ("attention_ctx_grad_fwd_tc", "attention_ctx_grad_fwd", lambda: (_attn(BF16, False), dict(use_tc=True))),
    ("attention_ctx_grad_fwd_simt_ragged", "attention_ctx_grad_fwd",
     lambda: (_attn(F32, False, ragged=True), dict(use_tc=False))),
    ("attention_ctx_bwd_tc_ragged", "attention_ctx_bwd", lambda: (_attn(BF16, True, ragged=True), dict(use_tc=True))),
    ("attention_ctx_bwd_simt_n0", "attention_ctx_bwd", lambda: (_attn(F32, True, n=0), dict(use_tc=False))),
    ("embed_input_bwd", "embed_input_bwd",
     lambda: ((t(12, 16, dtype=BF16), t(16, 3), t(16), t(12, 3), t(12), 4, 3, 3, 16, 2), {})),
    ("embed_input_bwd_ragged", "embed_input_bwd",
     lambda: ((t(12, 16), t(16, 9), t(16), t(12, 9), t(12), 4, 3, 9, 16, 4, t(3, dtype=I32)), {})),
]


class FakeLib:
    def __init__(self):
        self.calls, self.names = [], {}
        for name in LIG._PROTOTYPES:
            setattr(self, name, self._entry(name))

    def _ptr(self, v):
        return self.names.get(v, "<not an argument>" if v else None)

    def _struct(self, d):
        out = {}
        for field, ctype in d._fields_:
            v = getattr(d, field)
            if isinstance(v, ctypes.Structure):
                out[field] = self._struct(v)
            elif ctype is ctypes.c_void_p:
                out[field] = self._ptr(v)
            else:
                out[field] = v
        return out

    def _arg(self, a):
        if a is STREAM:
            return "<stream>"
        if isinstance(a, ctypes.c_void_p):
            return self._ptr(a.value)
        if hasattr(a, "_obj"):
            return {"byref": self._struct(a._obj)}
        return a

    def _entry(self, name):
        def f(*args):
            self.calls.append({"fn": name, "args": [self._arg(a) for a in args]})
            return 0
        return f


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(L, "load", lambda: lib)
    monkeypatch.setattr(L, "stream_ptr", lambda device=None: STREAM)
    return lib


def _record(case, lib, monkeypatch):
    _, wrapper, build = next(c for c in CASES if c[0] == case)
    fn = getattr(LIG, wrapper)
    args, kwargs = build()
    bound = inspect.signature(fn).bind(*args, **kwargs).arguments
    names = {id(v): k for k, v in bound.items() if torch.is_tensor(v)}
    lib.names = {v.data_ptr(): f"{k}+0" for k, v in bound.items() if torch.is_tensor(v)}
    checked = set()
    monkeypatch.setattr(L, "require_cuda",
                        lambda *ts: checked.update(names[id(x)] for x in ts if x is not None and id(x) in names))
    lib.calls = []
    n0 = L.launch_count()
    fn(*args, **kwargs)
    return {"calls": lib.calls, "launches": L.launch_count() - n0, "require_cuda": sorted(checked)}


@pytest.mark.parametrize("case", [c[0] for c in CASES])
def test_call_log_matches_golden(case, fake, monkeypatch):
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert list(golden) == [c[0] for c in CASES]
    assert _record(case, fake, monkeypatch) == golden[case]


@pytest.mark.parametrize("case", [c[0] for c in CASES])
def test_cpu_tensor_is_rejected_before_the_library_is_called(case, fake):
    """Each tensor argument in turn on the CPU, the others on a CUDA device (unbacked): require_cuda's error, no call, no
    launch."""
    from torch._subclasses.fake_tensor import FakeTensorMode
    _, wrapper, build = next(c for c in CASES if c[0] == case)
    fn = getattr(LIG, wrapper)
    args, kwargs = build()
    with FakeTensorMode():
        conv = lambda a: torch.empty_strided(a.shape, a.stride(), dtype=a.dtype, device="cuda") if torch.is_tensor(a) else a
        cuda_args = [conv(a) for a in args]
        cuda_kwargs = {k: conv(v) for k, v in kwargs.items()}
    probes = [("a", i) for i, a in enumerate(args) if torch.is_tensor(a)]
    probes += [("k", k) for k, v in kwargs.items() if torch.is_tensor(v)]
    for where, i in probes:
        a, kw = list(cuda_args), dict(cuda_kwargs)
        if where == "a":
            a[i] = args[i]
        else:
            kw[i] = kwargs[i]
        fake.calls = []
        n0 = L.launch_count()
        with pytest.raises(RuntimeError, match="sm_90a CUDA kernels only"):
            fn(*a, **kw)
        assert fake.calls == [] and L.launch_count() == n0, (case, i)


def test_wrong_key_count_tensor_is_rejected(fake, monkeypatch):
    monkeypatch.setattr(L, "require_cuda", lambda *ts: None)
    n0 = L.launch_count()
    args = _attn(F32, False)
    args[-1] = t(2, dtype=torch.int64)
    with pytest.raises(TypeError, match="int32"):
        LIG.attention_ctx_grad_fwd(*args, use_tc=False)
    args = _attn(BF16, True)
    args[-1] = t(3, dtype=I32)
    with pytest.raises(TypeError, match=r"\(2,\)"):
        LIG.attention_ctx_bwd(*args, use_tc=True)
    with pytest.raises(TypeError, match=r"\(3,\)"):
        LIG.embed_input_bwd(t(12, 16), t(16, 3), t(16), t(12, 3), t(12), 4, 3, 3, 16, 4, t(2, dtype=I32))
    assert fake.calls == [] and L.launch_count() == n0


def write_golden():
    mp = pytest.MonkeyPatch()
    try:
        lib = FakeLib()
        mp.setattr(L, "load", lambda: lib)
        mp.setattr(L, "stream_ptr", lambda device=None: STREAM)
        log = {c[0]: _record(c[0], lib, mp) for c in CASES}
    finally:
        mp.undo()
    with open(GOLDEN, "w") as f:
        json.dump(log, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    write_golden()
