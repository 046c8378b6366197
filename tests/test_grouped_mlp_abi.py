"""The row-grouped layer's C entry points: declared as plain C99, and their argument checks run without a GPU."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_grouped_declarations_compile_as_c99_and_link(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    from scanobjectnn_b200.build import build_library
    build_library()
    src = tmp_path / "use_grouped.c"
    src.write_text('#include "psa.h"\n#include <stddef.h>\n'
                   "int main(void) {\n"
                   "    int (*f0)(long long, long long, const float*, const psa_mlp*, const float*, float*, void*, size_t, psa_stream_t) =\n"
                   "        psa_shared_mlp_grouped;\n"
                   "    int (*f1)(long long, long long, int, int, const psa_act_in*, const float*, const float*, const float*, float*, float*,\n"
                   "              void*, size_t, psa_stream_t) = psa_train_dense_fwd_grouped;\n"
                   "    int (*f2)(long long, long long, int, const psa_grad_in*, float*, psa_stream_t) = psa_train_bias_grad_grouped;\n"
                   "    return (f0 != NULL && f1 != NULL && f2 != NULL) ? 0 : 1;\n}\n")
    inc = os.path.join(ROOT, "include")
    libdir = os.path.join(ROOT, "scanobjectnn_b200")
    exe = tmp_path / "use_grouped"
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", inc, str(src), "-L", libdir, "-lpsa", f"-Wl,-rpath,{libdir}", "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([str(exe)]).returncode == 0


def test_group_rows_that_do_not_divide_rows_are_rejected():
    from scanobjectnn_b200 import _lib
    lib = _lib.load()
    fake = C.c_void_p(16)          # never dereferenced: the checks fail before anything is launched
    mlp = _lib.PsaMlp()
    mlp.n_layers = 1
    mlp.channels[0], mlp.channels[1] = 64, 128
    mlp.weight[0] = mlp.shift[0] = 16
    ain, gin = _lib.PsaActIn(x=16, ld=64), _lib.PsaGradIn()
    ws = C.c_size_t(0)
    for rows, group_rows in ((10, 3), (10, 0), (10, -2)):
        assert lib.psa_shared_mlp_grouped(rows, group_rows, fake, C.byref(mlp), fake, fake, fake, ws, None) == -1
        assert b"group_rows" in lib.psa_last_error()
        assert lib.psa_train_dense_fwd_grouped(rows, group_rows, 64, 128, C.byref(ain), fake, None, fake, fake, None, None, ws, None) == -1
        assert lib.psa_train_bias_grad_grouped(rows, group_rows, 128, C.byref(gin), fake, None) == -1
    # a missing group input is an invalid argument too
    assert lib.psa_shared_mlp_grouped(12, 3, fake, C.byref(mlp), None, fake, fake, ws, None) == -1
    assert lib.psa_train_dense_fwd_grouped(12, 3, 64, 128, C.byref(ain), fake, None, None, fake, None, None, ws, None) == -1
