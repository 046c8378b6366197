"""The C-ABI library loads and exports every symbol include/psa.h declares; header, ctypes table and ELF agree.
No compute calls (runs without a GPU)."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    text = open(os.path.join(ROOT, "include", "psa.h")).read()
    return sorted(set(re.findall(r"PSA_API\s+[\w\s\*]+?\b(psa_\w+)\s*\(", text)))


def test_library_builds_and_exports_header_symbols():
    from scanobjectnn_b200 import _lib
    from scanobjectnn_b200.build import build_library
    path = build_library()
    out = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (psa_\w+)", out))
    declared = _header_symbols()
    assert len(declared) >= 25
    missing = [s for s in declared if s not in exported]
    assert not missing, f"declared in psa.h but not exported: {missing}"
    extra = sorted(exported - set(declared))
    assert not extra, f"exported but not declared in psa.h: {extra}"
    lib = _lib.load()
    for s in declared:
        assert hasattr(lib, s)
    assert set(_lib.SIGNATURES) | set(_lib.INFO_SYMBOLS) == set(declared)
    assert lib.psa_version() >= 100 and lib.psa_sm_arch() == 90


def test_library_is_sm90a_only_and_uses_tensor_cores():
    from scanobjectnn_b200.build import LIB, build_library
    build_library()
    elf = subprocess.run(["cuobjdump", "-lelf", LIB], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", elf))
    assert archs == {"90a"}, archs
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    assert "HGMMA" in sass and "UBLKCP" in sass     # wgmma.mma_async / cp.async.bulk


def test_invalid_arguments_are_rejected_without_a_gpu():
    from scanobjectnn_b200 import _lib
    lib = _lib.load()
    null = C.c_void_p(0)
    assert lib.psa_farthest_point_sample(2, 0, 4, null, null, null, null) == -1        # n = 0 with m > 0
    assert b"at least one" in lib.psa_last_error()
    assert lib.psa_farthest_point_sample(-1, 8, 4, null, null, null, null) == -1
    assert lib.psa_query_ball_point(1, 8, 4, C.c_float(0.2), -3, null, null, null, null, null) == -1
    assert lib.psa_farthest_point_sample(0, 8, 4, null, null, null, null) == 0         # b = 0: no-op
    assert lib.psa_set_mlp_mode(5) == -1 and lib.psa_set_mlp_mode(-1) == -1


def test_ops_refuse_cpu_tensors():
    import torch

    from scanobjectnn_b200 import ops
    with pytest.raises(RuntimeError):
        ops.farthest_point_sample(4, torch.zeros((1, 8, 3)))
    with pytest.raises(RuntimeError):
        ops.query_ball_point(0.2, 4, torch.zeros((1, 8, 3)), torch.zeros((1, 2, 3)))


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "scanobjectnn_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, re.M), f
                assert "liboracle" not in text and "oracle/_ref" not in text, f


def test_header_is_plain_c99_and_links_from_c(tmp_path):
    """The boundary is a C ABI: include/psa.h compiles as C99 (no C++, no torch types) and a C program links against libpsa.so."""
    import shutil
    import subprocess

    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    src = tmp_path / "use_psa.c"
    src.write_text('#include "psa.h"\n#include <stddef.h>\n'
                   "int main(void) {\n"
                   "    /* taking the addresses forces the prototypes to resolve at link time; nothing is launched */\n"
                   "    void* f[] = {(void*)psa_farthest_point_sample, (void*)psa_query_ball_point, (void*)psa_sa_module_infer, (void*)psa_sa_conv1_prebn,\n"
                   "                 (void*)psa_three_nn_interpolate, (void*)psa_knn_graph, (void*)psa_last_error};\n"
                   "    return (f[0] != NULL && psa_get_mlp_mode() >= 0) ? 0 : 1;\n}\n")
    inc = os.path.join(ROOT, "include")
    libdir = os.path.join(ROOT, "scanobjectnn_b200")
    exe = tmp_path / "use_psa"
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", inc, str(src), "-L", libdir, "-lpsa", f"-Wl,-rpath,{libdir}", "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
