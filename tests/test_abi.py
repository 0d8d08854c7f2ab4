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


def test_version_and_arch():
    l = _lib.lib()
    assert l.orp_version() >= 100
    assert l.orp_compiled_sm() == 90


def test_sass_is_sm90a_only():
    import subprocess
    out = subprocess.run(["cuobjdump", "--list-elf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs
