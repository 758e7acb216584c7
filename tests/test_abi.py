"""CPU-side checks of the C-ABI boundary: the in-tree library loads and exports every symbol that
include/dlrm_b200.h declares (no compute calls: there is no GPU here)."""
import os
import re

from dlrm_b200 import _build, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "dlrm_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dlrm_b200_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = _lib.lib()
    syms = header_symbols()
    assert len(syms) >= 13
    for s in syms:
        assert hasattr(lib, s), "libdlrm_b200.so does not export " + s
    assert sorted(_lib.SYMBOLS) == syms, "dlrm_b200/_lib.py and the header disagree"


def test_abi_version_and_error_text():
    lib = _lib.lib()
    assert lib.dlrm_b200_abi_version() == 1
    # argument validation happens before any CUDA call -> testable without a device
    rc = lib.dlrm_b200_emb_bag_fwd(None, 1000, 128, 1, 8, 0, None, 0, 0, None)
    assert rc != 0
    assert b"num_tables" in lib.dlrm_b200_last_error()


def test_built_for_sm90a_only():
    cuobjdump = os.path.join(os.path.dirname(_build.nvcc_path()), "cuobjdump")
    out = os.popen("%s -lelf %s 2>/dev/null" % (cuobjdump, _build.LIB)).read()
    assert "sm_90a" in out
    assert "sm_100" not in out and "sm_80" not in out


def test_product_does_not_import_oracle():
    """The oracle is the checker: nothing under dlrm_b200/ may import or execute it."""
    pkg = os.path.join(ROOT, "dlrm_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), f


def test_struct_layouts_match_the_header(tmp_path):
    """sizeof / offsetof of every struct in include/dlrm_b200.h, as a C compiler sees them, equal the
    ctypes mirrors in dlrm_b200/_lib.py (field names are the header's)."""
    import ctypes as C
    import subprocess

    pairs = {"dlrm_emb_fwd_table_t": _lib.EmbFwdTable, "dlrm_emb_bwd_table_t": _lib.EmbBwdTable,
             "dlrm_emb_dedup_t": _lib.EmbDedup, "dlrm_gemm_tc_desc_t": _lib.GemmTcDesc,
             "dlrm_dense_layer_t": _lib.DenseLayer}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "dlrm_b200.h"', "int main(void) {"]
    for cname, cls in pairs.items():
        lines.append('printf("%s %%zu\\n", sizeof(%s));' % (cname, cname))
        for fname, _ in cls._fields_:
            lines.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (cname, fname, cname, fname))
    lines += ["return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe], check=True)
    got = dict(l.split() for l in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines())
    for cname, cls in pairs.items():
        assert int(got[cname]) == C.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert int(got[cname + "." + fname]) == getattr(cls, fname).offset, cname + "." + fname


def test_library_freshness_does_not_depend_on_where_the_tree_lives(tmp_path, monkeypatch):
    """The in-tree library is built in one place and run from a copy of the tree under another path (the GPU box): the
    freshness digest must cover the sources' contents and names, not their absolute paths -- otherwise every first
    process of a copy rebuilds the library, all ranks of a torchrun at once."""
    import shutil

    from dlrm_b200 import _build

    want = _build._digest()
    root = tmp_path / "elsewhere"
    shutil.copytree(_build.CSRC, root / "dlrm_b200" / "csrc")
    shutil.copytree(os.path.join(os.path.dirname(_build.HERE), "include"), root / "include")
    monkeypatch.setattr(_build, "HERE", str(root / "dlrm_b200"))
    monkeypatch.setattr(_build, "CSRC", str(root / "dlrm_b200" / "csrc"))
    assert _build._digest() == want
    with open(root / "dlrm_b200" / "csrc" / "api.cu", "a") as fh:
        fh.write("\n// edited\n")
    assert _build._digest() != want
