"""CPU-only: liborx.so loads, exports exactly the symbols include/orx.h declares, and refuses to
compute without a device (no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    from openrec_b200 import build
    return build.build()


def _declared():
    src = open(os.path.join(ROOT, "include", "orx.h")).read()
    return sorted(set(re.findall(r"ORX_API\s+(?:const\s+char\*|int)\s+(orx_\w+)\s*\(", src)))


def test_header_symbols_exported(built):
    out = subprocess.run(["nm", "-D", "--defined-only", built], capture_output=True, text=True, check=True).stdout
    exported = sorted(set(re.findall(r"\sT\s+(orx_\w+)", out)))
    assert _declared() == exported


def test_ctypes_signatures_cover_header(built):
    from openrec_b200 import _lib
    assert sorted(_lib.SIGNATURES) == _declared()
    l = _lib.lib()
    assert l.orx_abi_version() == 1


def _prototypes():
    """name -> list of parameter declarations of every ORX_API prototype in include/orx.h."""
    src = re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", "orx.h")).read(), flags=re.S)
    out = {}
    for name, params in re.findall(r"ORX_API\s+(?:const\s+char\*|int)\s+(orx_\w+)\s*\(([^;]*?)\)\s*;", src, flags=re.S):
        params = " ".join(params.split())
        out[name] = [] if params in ("", "void") else [p.strip() for p in params.split(",")]
    return out


def test_ctypes_argument_lists_match_header(built):
    """Every binding has as many arguments as its prototype, and pointer / integer / float kinds agree position by
    position (a parameter added to orx.h but not to _lib.SIGNATURES would shift every later argument silently)."""
    from openrec_b200 import _lib
    protos = _prototypes()
    assert sorted(protos) == sorted(_lib.SIGNATURES)

    def kind_c(decl):
        if "*" in decl or re.search(r"\borx_(handle|stream)_t\b", decl):
            return "ptr"
        if re.search(r"\b(float|double)\b", decl):
            return "float"
        return "int"

    def kind_py(t):
        if t in (C.c_float, C.c_double):
            return "float"
        if t in (C.c_void_p, C.c_char_p) or hasattr(t, "_type_") and not isinstance(t._type_, str):
            return "ptr"
        return "int"

    for name, params in protos.items():
        sig = _lib.SIGNATURES[name]
        assert len(sig) == len(params), f"{name}: header has {len(params)} parameters, _lib.SIGNATURES {len(sig)}"
        for k, (decl, t) in enumerate(zip(params, sig)):
            assert kind_c(decl) == kind_py(t), f"{name} argument {k}: '{decl}' vs {t}"


def test_sm90a_only(built):
    out = subprocess.run(["cuobjdump", "--list-elf", built], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_no_cpu_fallback(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("device present")
    from openrec_b200 import _lib, native
    h = C.c_void_p()
    rc = _lib.lib().orx_create(0, C.byref(h))
    assert rc != 0 and not h.value
    assert _lib.last_error()
    with pytest.raises(RuntimeError):
        native.engine()
