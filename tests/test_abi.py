"""CPU-side checks of the drop-in boundary: the C-ABI library builds, loads and exports exactly the
entry points include/clipbert_b200.h declares (no compute calls: there is no GPU here)."""
import ctypes
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "clipbert_b200.h")


def _declared():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(cb_[a-z0-9_]+)\s*\(", text)))


def test_library_builds_and_exports_every_declared_symbol():
    from clipbert_b200 import build
    path = build.build()
    assert os.path.exists(path)
    lib = ctypes.CDLL(path)
    names = _declared()
    assert len(names) >= 24
    for n in names:
        assert hasattr(lib, n), "header declares %s but the library does not export it" % n
    exported = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True).stdout
    extra = set(re.findall(r" T (cb_[a-z0-9_]+)", exported)) - set(names)
    assert not (extra - {"cb_debug_gemm_timeline", "cb_debug_gemm_kch", "cb_debug_gemm_sm_limit", "cb_debug_gemm_occ2", "cb_debug_gemm_mn3d", "cb_debug_attention_general", "cb_debug_attention_flash", "cb_debug_attention_rows48", "cb_debug_attention_flash_pipe"}), "exported but undeclared: %s" % sorted(extra)


def test_header_compiles_as_plain_c(tmp_path):
    src = tmp_path / "t.c"
    src.write_text('#include "clipbert_b200.h"\nint main(void) { cb_gemm_desc d; (void)d; return sizeof(d) > 0 ? 0 : 1; }\n')
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src), "-o",
                        str(tmp_path / "t.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_ctypes_struct_matches_c_layout(tmp_path):
    from clipbert_b200 import _lib
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "clipbert_b200.h"\n'
                   'int main(void){printf("%zu %zu %zu %zu %zu\\n", sizeof(cb_gemm_desc), offsetof(cb_gemm_desc, a), '
                   'offsetof(cb_gemm_desc, scale), offsetof(cb_gemm_desc, out), offsetof(cb_gemm_desc, dropout_seed));return 0;}\n')
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    c = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()]
    D = _lib.GemmDesc
    assert c == [ctypes.sizeof(D), D.a.offset, D.scale.offset, D.out.offset, D.dropout_seed.offset]


def test_status_and_version_calls_work_without_a_gpu():
    from clipbert_b200 import _lib
    lib = _lib.lib()
    assert lib.cb_version() == 100 and lib.cb_sm_arch() == 90
    assert lib.cb_launch_count() >= 0
    d = _lib.GemmDesc()
    assert lib.cb_gemm(ctypes.byref(d), None) == -1          # CB_ERR_INVALID, no kernel launched
    assert b"null operand" in lib.cb_last_error()


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "clipbert_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, flags=re.M), f
                assert "torch.nn.functional" not in text or f == "modeling.py", f   # F.* only in the loss glue
