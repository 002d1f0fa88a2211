"""The ctypes binding (_lib.py) against the C ABI it restates (include/pfn_b200.h).

On the host, without the built library: every ctypes Structure has the member names, kinds, offsets and size of its
header struct (as the host C compiler lays it out), every mirrored enum constant has the header's value, and every
`_PROTOTYPES` entry has the parameter kinds of its prototype.  With the built library: it loads on a CPU-only box and
exports every symbol the header declares."""
import ctypes
import os
import re
import shutil
import subprocess
import types

import pytest

from transformerscandobayesianinference_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C_TYPES = {"int": ctypes.c_int, "uint32_t": ctypes.c_uint32, "float": ctypes.c_float, "double": ctypes.c_double,
           "long long": ctypes.c_longlong}


def _header():
    text = open(os.path.join(ROOT, "include", "pfn_b200.h")).read()
    return re.sub(r"/\*.*?\*/", "", text, flags=re.S)


def _declared_symbols():
    return sorted(set(re.findall(r"\b(pfn_[a-z0-9_]+)\s*\(", _header())))


def _ctype(decl):
    """The C type of a declaration `type name` with its spacing normalised ("const void* A" -> "const void*")."""
    return re.sub(r"\s*\*", "*", " ".join(re.fullmatch(r"\s*(.*?[\s*])\w+\s*", decl, flags=re.S).group(1).split()))


def _structs():
    """{tag: [(member, C type), ...]} of every `typedef struct pfn_* {...}`, members in declaration order."""
    out = {}
    for tag, body in re.findall(r"typedef\s+struct\s+(pfn_\w+)\s*\{(.*?)\}", _header(), flags=re.S):
        members = []
        for decl in filter(str.strip, body.split(";")):
            first, *more = decl.split(",")                  # int M, N, K;
            ctype = _ctype(first)
            members += [(first.split()[-1].lstrip("*"), ctype)] + [(n.strip(), ctype) for n in more]
        out[tag] = members
    return out


def _mirrors():
    """{tag: ctypes Structure of _lib.py}: GemmDesc mirrors pfn_gemm_desc, AdamTensor pfn_adam_tensor."""
    return {"pfn_" + re.sub(r"(?<!^)(?=[A-Z])", "_", name).lower(): cls for name, cls in vars(L).items()
            if isinstance(cls, type) and issubclass(cls, ctypes.Structure) and cls.__module__ == L.__name__}


def _enums():
    """The PFN_* names of every enum of the header, one list per enum."""
    return [re.findall(r"\b(PFN_\w+)\s*=", body) for body in re.findall(r"\benum\s*\{(.*?)\}", _header(), flags=re.S)]


def _prototypes():
    """{name: (return C type, [parameter declarations])} of every entry point; `(void)` has no parameters."""
    out = {}
    for chunk in _header().split(";"):
        m = re.fullmatch(r"\s*([^{}()#]*?)\s*\b(pfn_\w+)\s*\(([^()]*)\)\s*", chunk)
        if m:
            out[m.group(2)] = (_ctype(m.group(1) + " x"), [p for p in m.group(3).split(",") if p.strip() != "void"])
    return out


def _argtype(param, mirrors):
    """The ctypes type a parameter declaration binds to."""
    ctype = _ctype(param)
    desc = re.fullmatch(r"const (pfn_\w+_desc)\*", ctype)
    if desc:
        return ctypes.POINTER(mirrors[desc.group(1)])
    return ctypes.c_void_p if ctype.endswith("*") else C_TYPES[ctype]


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """{("sizeof", tag) / ("offsetof", tag, member) / ("enum", name): value} as the host C compiler sees the header."""
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler (cc / gcc)")
    lines = []
    for tag, members in _structs().items():
        lines.append(f'printf("sizeof {tag} %zu\\n", sizeof({tag}));')
        lines += [f'printf("offsetof {tag} {m} %zu\\n", offsetof({tag}, {m}));' for m, _ in members]
    lines += [f'printf("enum {e} %lld\\n", (long long){e});' for block in _enums() for e in block]
    tmp = tmp_path_factory.mktemp("cabi")
    src, exe = tmp / "layout.c", tmp / "layout"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "pfn_b200.h"\n\nint main(void) {\n'
                   + "".join(f"  {s}\n" for s in lines) + "  return 0;\n}\n")
    r = subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    return {tuple(line.split()[:-1]): int(line.split()[-1]) for line in out.splitlines()}


def test_struct_layouts_match_header(compiled):
    structs, mirrors = _structs(), _mirrors()
    assert set(mirrors) == set(structs) and len(structs) >= 9
    for tag, members in structs.items():
        cls = mirrors[tag]
        assert [n for n, _ in cls._fields_] == [n for n, _ in members], tag
        for (name, ctype), (_, t) in zip(members, cls._fields_):
            ok = (t is ctypes.c_void_p or issubclass(t, ctypes._Pointer)) if ctype.endswith("*") else t is C_TYPES[ctype]
            assert ok, f"{tag}.{name}: {ctype} mirrored as {t.__name__}"
            assert getattr(cls, name).offset == compiled["offsetof", tag, name], f"{tag}.{name}"
        assert ctypes.sizeof(cls) == compiled["sizeof", tag], tag


def test_constants_match_header(compiled):
    mirrored = [e for block in _enums() for e in block if hasattr(L, e[len("PFN_"):])]
    assert len(mirrored) >= 30
    for e in mirrored:
        assert getattr(L, e[len("PFN_"):]) == compiled["enum", e], e


def test_gp_mcmc_diag_names_follow_header(compiled):
    block = next(b for b in _enums() if "PFN_GP_MCMC_NDIAG" in b)
    cols = sorted((e for e in block if e != "PFN_GP_MCMC_NDIAG"), key=lambda e: compiled["enum", e])
    assert [compiled["enum", e] for e in cols] == list(range(len(cols)))
    assert L.GP_MCMC_DIAG_NAMES == tuple(e[len("PFN_GP_MCMC_"):].lower() for e in cols)
    assert len(L.GP_MCMC_DIAG_NAMES) == compiled["enum", "PFN_GP_MCMC_NDIAG"]


def test_prototypes_match_header():
    protos, mirrors = _prototypes(), _mirrors()
    assert set(L._PROTOTYPES) == set(protos) == set(_declared_symbols())
    for name, (_, params) in protos.items():
        assert list(L._PROTOTYPES[name]) == [_argtype(p, mirrors) for p in params], name


def test_declare_applies_the_table():
    protos = _prototypes()
    lib = types.SimpleNamespace(**{name: types.SimpleNamespace() for name in protos})
    assert L.declare(lib) is lib
    for name, (ret, _) in protos.items():
        fn = getattr(lib, name)
        assert fn.restype is {"int": ctypes.c_int, "const char*": ctypes.c_char_p}[ret], name
        assert fn.argtypes == L._PROTOTYPES[name]
    del lib.pfn_knn_cv
    with pytest.raises(RuntimeError, match="does not export pfn_knn_cv"):
        L.declare(lib)


def test_header_symbols_are_exported():
    lib = L.load()
    declared = _declared_symbols()
    assert len(declared) >= 15
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/pfn_b200.h but not exported"
    assert set(L.EXPORTED_SYMBOLS) == set(declared)


def test_version_and_error_string():
    lib = L.load()
    assert lib.pfn_version() == 1
    d = L.GemmDesc()
    rc = lib.pfn_gemm_simt(ctypes.byref(d), None)       # argument validation happens before any CUDA call
    assert rc != 0 and b"empty problem" in lib.pfn_last_error()
    a = L.AttnDesc()
    assert lib.pfn_attention_fwd_tc(ctypes.byref(a), None) != 0
