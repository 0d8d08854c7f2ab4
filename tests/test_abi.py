"""CPU: the C-ABI library loads and exports every symbol include/orp_b200.h declares
(no compute calls - there is no GPU here)."""
import os
import re

from orientedreppoints_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "orp_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(orp_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    l = _lib.lib()
    names = _declared()
    assert len(names) >= 12
    for n in names:
        assert hasattr(l, n), n
        assert n in _lib.SIGNATURES, "binding missing for %s" % n
    assert sorted(_lib.SIGNATURES) == names


def test_bindings_match_declared_arity():
    """every binding passes as many arguments as the header declares: a parameter added to a declaration (a stream, say)
    and not to _lib.SIGNATURES would make ctypes pass garbage in its place"""
    src = open(os.path.join(ROOT, "include", "orp_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    decls = dict(re.findall(r"\b(orp_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src))
    assert sorted(decls) == _declared()
    for name, params in decls.items():
        params = params.strip()
        n = 0 if params in ("", "void") else params.count(",") + 1
        assert len(_lib.SIGNATURES[name][1]) == n, (name, n, len(_lib.SIGNATURES[name][1]))


def test_version_and_arch():
    l = _lib.lib()
    assert l.orp_version() >= 100
    assert l.orp_compiled_sm() == 90


def test_sass_is_sm90a_only():
    import subprocess
    out = subprocess.run(["cuobjdump", "--list-elf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_rnms_plan_record_matches_header():
    """orp_rnms_last_plan is declared, exported and bound, and RnmsPlan has the header's fields in the header's order"""
    import ctypes
    assert "orp_rnms_last_plan" in _declared()
    assert hasattr(_lib.lib(), "orp_rnms_last_plan")
    src = open(os.path.join(ROOT, "include", "orp_b200.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} orp_rnms_plan;", src).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        m = re.match(r"\s*(int32_t|int64_t)\s+(.*)", decl, flags=re.S)
        if m:
            fields += [(n.strip(), m.group(1)) for n in m.group(2).split(",")]
    want = {"int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64}
    assert [(n, want[t]) for n, t in fields] == list(_lib.RnmsPlan._fields_)
    assert ctypes.sizeof(_lib.RnmsPlan) == 64
