"""The ragged-attention binding (_lib_ragged.py) against its header (include/pfn_b200_ragged.h), on the host.

Without the built library: each ctypes Structure has the member names, kinds, offsets and size of its header struct as
the host C compiler lays it out, `_PROTOTYPES` has every prototype's parameter kinds, and every wrapper's calls match the
log in tests/golden/lib_calls_ragged.json (entry points in order, descriptors field by field with pointers as the name of
the argument tensor they point into, launches counted, tensors checked), recorded against a fake of the library
(`python tests/test_ragged_cabi_host.py` rewrites it).  A CPU tensor in any argument is rejected before the library is
called.  With the built library: it exports every entry point the header declares."""
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

from transformerscandobayesianinference_b200 import _lib as L, _lib_ragged as LR  # noqa: E402

HEADER = os.path.join(ROOT, "include", "pfn_b200_ragged.h")
GOLDEN = os.path.join(ROOT, "tests", "golden", "lib_calls_ragged.json")
C_TYPES = {"int": ctypes.c_int, "float": ctypes.c_float}
MIRRORS = {"pfn_attn_ragged_desc": LR.AttnRaggedDesc, "pfn_attn_ctx_ragged_desc": LR.AttnCtxRaggedDesc}
BF16, F32, I32 = torch.bfloat16, torch.float32, torch.int32
STREAM = object()


def t(*shape, dtype=F32):
    return torch.zeros(shape, dtype=dtype)


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def _ctype(decl):
    return re.sub(r"\s*\*", "*", " ".join(re.fullmatch(r"\s*(.*?[\s*])\w+\s*", decl, flags=re.S).group(1).split()))


def _structs():
    out = {}
    for tag, body in re.findall(r"typedef\s+struct\s+(pfn_\w+)\s*\{(.*?)\}", _header(), flags=re.S):
        members = []
        for decl in filter(str.strip, body.split(";")):
            first, *more = decl.split(",")
            ctype = _ctype(first)
            members += [(first.split()[-1].lstrip("*"), ctype)] + [(n.strip(), ctype) for n in more]
        out[tag] = members
    return out


def _prototypes():
    out = {}
    for chunk in _header().split(";"):
        m = re.fullmatch(r"\s*([^{}()#]*?)\s*\b(pfn_\w+)\s*\(([^()]*)\)\s*", chunk)
        if m:
            out[m.group(2)] = [p for p in m.group(3).split(",") if p.strip() != "void"]
    return out


def test_struct_layouts_match_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler (cc / gcc)")
    structs = _structs()
    assert set(structs) == set(MIRRORS)
    lines = []
    for tag, members in structs.items():
        lines.append(f'printf("sizeof {tag} %zu\\n", sizeof({tag}));')
        lines += [f'printf("offsetof {tag} {m} %zu\\n", offsetof({tag}, {m}));' for m, _ in members]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "pfn_b200_ragged.h"\n\nint main(void) {\n'
                   + "".join(f"  {s}\n" for s in lines) + "  return 0;\n}\n")
    r = subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    compiled = {tuple(line.split()[:-1]): int(line.split()[-1]) for line in out.splitlines()}
    for tag, members in structs.items():
        cls = MIRRORS[tag]
        assert [n for n, _ in cls._fields_] == [n for n, _ in members], tag
        for (name, ctype), (_, ty) in zip(members, cls._fields_):
            assert ty is ctypes.c_void_p if ctype.endswith("*") else ty is C_TYPES[ctype], f"{tag}.{name}"
            assert getattr(cls, name).offset == compiled["offsetof", tag, name], f"{tag}.{name}"
        assert ctypes.sizeof(cls) == compiled["sizeof", tag], tag


def test_prototypes_match_header():
    protos = _prototypes()
    assert list(LR._PROTOTYPES) == list(protos) and len(protos) == 4
    for name, params in protos.items():
        tag = re.fullmatch(r"const (pfn_\w+_desc)\*", _ctype(params[0])).group(1)
        assert LR._PROTOTYPES[name] == [ctypes.POINTER(MIRRORS[tag]), ctypes.c_void_p], name
        assert _ctype(params[1]) == "void*"


def test_declare_checks_every_symbol():
    class Fake:
        pass
    lib = Fake()
    for name in LR._PROTOTYPES:
        setattr(lib, name, Fake())
    assert LR.declare(lib) is lib
    assert lib.pfn_attention_ragged_fwd_tc.restype is ctypes.c_int
    del lib.pfn_attention_ctx_ragged_fwd_tc
    with pytest.raises(RuntimeError, match="does not export pfn_attention_ctx_ragged_fwd_tc"):
        LR.declare(lib)


def test_header_symbols_are_exported():
    lib = L.load()
    for name in LR.EXPORTED_SYMBOLS:
        assert hasattr(lib, name), f"{name} declared in include/pfn_b200_ragged.h but not exported"


# ---- the wrappers against a recording fake of the library ----------------------------------------------------------
CASES = [
    ("attention_ragged_fwd_tc", "attention_ragged_fwd",
     lambda: ((t(16, 24, dtype=BF16), t(16, 8, dtype=BF16), 8, 2, 2, 4, t(2, dtype=I32)), dict(use_tc=True))),
    ("attention_ragged_fwd_simt", "attention_ragged_fwd",
     lambda: ((t(16, 24), t(16, 8), 8, 2, 2, 4, t(2, dtype=I32)), dict(use_tc=False))),
    ("attention_ctx_ragged_fwd_tc", "attention_ctx_ragged_fwd",
     lambda: ((t(8, 24, dtype=BF16), t(6, 16, dtype=BF16), t(8, 8, dtype=BF16), 4, 3, 2, 2, 4, t(2, dtype=I32)),
              dict(use_tc=True))),
    ("attention_ctx_ragged_fwd_simt", "attention_ctx_ragged_fwd",
     lambda: ((t(8, 24), t(6, 16), t(8, 8), 4, 3, 2, 2, 4, t(2, dtype=I32)), dict(use_tc=False))),
    ("attention_ctx_ragged_fwd_n0", "attention_ctx_ragged_fwd",
     lambda: ((t(8, 24, dtype=BF16), t(6, 16, dtype=BF16), t(8, 8, dtype=BF16), 4, 0, 2, 2, 4, t(2, dtype=I32)),
              dict(use_tc=True))),
]


class FakeLib:
    def __init__(self):
        self.calls, self.names = [], {}
        for name in LR._PROTOTYPES:
            setattr(self, name, self._entry(name))

    def _entry(self, name):
        def f(desc, stream):
            d = desc._obj
            fields = {}
            for field, ctype in d._fields_:
                v = getattr(d, field)
                fields[field] = self.names.get(v, "<not an argument>" if v else None) if ctype is ctypes.c_void_p else v
            self.calls.append({"fn": name, "args": [{"byref": fields}, "<stream>" if stream is STREAM else stream]})
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
    fn = getattr(LR, wrapper)
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
    launch.  An unread kv (n == 0) is not checked."""
    from torch._subclasses.fake_tensor import FakeTensorMode
    _, wrapper, build = next(c for c in CASES if c[0] == case)
    fn = getattr(LR, wrapper)
    args, kwargs = build()
    with FakeTensorMode():
        cuda_args = [torch.empty_strided(a.shape, a.stride(), dtype=a.dtype, device="cuda") if torch.is_tensor(a) else a
                     for a in args]
    probes = [i for i, a in enumerate(args) if torch.is_tensor(a) and not (case.endswith("_n0") and i == 1)]
    for i in probes:
        a = list(cuda_args)
        a[i] = args[i]
        fake.calls = []
        n0 = L.launch_count()
        with pytest.raises(RuntimeError, match="sm_90a CUDA kernels only"):
            fn(*a, **kwargs)
        assert fake.calls == [] and L.launch_count() == n0, (case, i)


def test_wrong_key_count_tensor_is_rejected(fake, monkeypatch):
    monkeypatch.setattr(L, "require_cuda", lambda *ts: None)
    with pytest.raises(TypeError, match="int32"):
        LR.attention_ragged_fwd(t(16, 24), t(16, 8), 8, 2, 2, 4, t(2, dtype=torch.int64), use_tc=False)
    with pytest.raises(TypeError, match=r"\(2,\)"):
        LR.attention_ctx_ragged_fwd(t(8, 24), t(6, 16), t(8, 8), 4, 3, 2, 2, 4, t(3, dtype=I32), use_tc=False)
    assert fake.calls == []


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
