"""The C-ABI library loads and exports every symbol include/editanything_b200.h declares, and the ctypes argument
structs have the header's layout."""
import os
import re

import pytest

from editanything_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _struct_members(name):
    """(member, array length or None) of `typedef struct <name> {...} <name>;` in the header, in declaration order."""
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "editanything_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), hdr, flags=re.S).group(1)
    members = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        for declarator in decl.split(","):
            member, length = re.search(r"(\w+)\s*(?:\[(\w+)\])?\s*$", declarator).groups()
            members.append((member, int(length) if length else None))
    return members


@pytest.mark.parametrize("struct,cls", [("ea_gemm_args", _lib.GemmArgs), ("ea_attn_args", _lib.AttnArgs),
                                        ("ea_gn_args", _lib.GnArgs)])
def test_ctypes_struct_matches_header(struct, cls):
    """A ctypes field missing, added or out of order shifts every later field: the library would read, say, the
    workspace pointer from where the caller stored a leading dimension."""
    fields = [(name, getattr(t, "_length_", None)) for name, t in cls._fields_]
    assert fields == _struct_members(struct)


def test_every_declared_symbol_is_exported_and_bound():
    hdr = open(os.path.join(ROOT, "include", "editanything_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(ea_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), f"{name} not exported by libea_b200.so"
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)


def test_nothing_is_exported_that_the_header_does_not_declare():
    """The reverse direction: no undeclared `ea_*` entry point (debug hooks exist only in -DEA_GEMM_TIMING builds)."""
    import shutil
    import subprocess
    nm = shutil.which("nm")
    if nm is None:
        import pytest
        pytest.skip("binutils nm not available")
    out = subprocess.run([nm, "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = {ln.split()[-1] for ln in out.splitlines() if ln.split() and ln.split()[-1].startswith("ea_")}
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "editanything_b200.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(ea_[a-z0-9_]+)\s*\(", hdr))
    assert exported <= declared, exported - declared


def test_library_reports_dtype_and_errors_without_gpu():
    lib = _lib.load()
    assert lib.ea_version() >= 1
    assert lib.ea_dtype_name() in (b"float16", b"bfloat16")
    assert b"argument" in lib.ea_strerror(-1)


def test_product_has_no_oracle_import():
    pkg = os.path.join(ROOT, "editanything_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f
