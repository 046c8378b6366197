"""Coordinate gradient of the fused first layer (psa_sa_conv1_bwd_xyz) without a GPU: argument rejection, and the SASS code shape of
its kernels (no float atomics -- every sum is added in a fixed order -- and no spills)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "scanobjectnn_b200", "libpsa.so")
XYZ_KERNELS = ("conv1_vxyz_kernel", "point_vsum_csr_kernel")


def _lib():
    from scanobjectnn_b200 import _lib
    from scanobjectnn_b200.build import build_library
    build_library()
    return _lib.load()


def test_conv1_bwd_xyz_rejects_bad_arguments():
    from scanobjectnn_b200._lib import PsaGradIn
    lib = _lib()
    null = C.c_void_p(0)
    fake = C.c_void_p(1 << 20)               # non-null, 16-byte aligned; never dereferenced: every check runs before a launch
    g = PsaGradIn()
    b, n, m, k = 2, 64, 16, 8
    need = lib.psa_sa_conv1_bwd_xyz_workspace_bytes(b, n, m, k)
    assert need >= b * m * k * 16 + b * (n + 1) * 4 + b * m * k * 4
    args = lambda C1, ws_bytes, w=fake: (b, n, m, k, C1, w, fake, C.byref(g), fake, fake, fake, C.c_size_t(ws_bytes), null)  # noqa: E731
    assert lib.psa_sa_conv1_bwd_xyz(0, n, m, k, 64, fake, fake, C.byref(g), fake, fake, fake, C.c_size_t(need), null) == -1
    assert lib.psa_sa_conv1_bwd_xyz(b, n, m, 0, 64, fake, fake, C.byref(g), fake, fake, fake, C.c_size_t(need), null) == -1
    assert lib.psa_sa_conv1_bwd_xyz(*args(64, need, w=null)) == -1                  # null weight
    assert b"null" in lib.psa_last_error()
    assert lib.psa_sa_conv1_bwd_xyz(*args(64, need, w=C.c_void_p((1 << 20) + 4))) == -1   # misaligned weight
    assert lib.psa_sa_conv1_bwd_xyz(*args(64, need - 4)) == -1                     # workspace too small
    assert b"workspace" in lib.psa_last_error()
    assert lib.psa_sa_conv1_bwd_xyz(*args(66, need)) == -2                         # C1 not a multiple of 4
    assert lib.psa_sa_conv1_bwd_xyz(*args(2048, need)) == -2                       # C1 above 1024


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_conv1_bwd_xyz_kernels_use_no_float_atomics():
    _lib()
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        mt = re.search(r"Function : (\S+)", line)
        if mt:
            name = mt.group(1) if any(kn in mt.group(1) for kn in XYZ_KERNELS) else None
            if name:
                funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    assert len(funcs) == 4, sorted(funcs)         # three lane-group widths of the row pass, one point pass
    for fn, lines in funcs.items():
        assert not any(re.search(r"\bRED\b|\bRED\.|\bATOM", l) for l in lines), f"{fn}: atomics"
        assert not any(re.search(r"\b(STL|LDL)\b", l) for l in lines), f"{fn}: local memory"


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not on PATH")
def test_conv1_bwd_xyz_kernels_do_not_spill(tmp_path):
    """ptxas -v on train.cu: the new kernels use no stack frame and spill nothing"""
    from scanobjectnn_b200 import build
    src = os.path.join(ROOT, "scanobjectnn_b200", "csrc", "train.cu")
    inc = [f"-I{os.path.join(ROOT, 'include')}", f"-I{os.path.join(ROOT, 'scanobjectnn_b200', 'csrc')}"]
    cmd = [shutil.which("nvcc"), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "train.o")] + inc
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    lines = res.stderr.splitlines()
    seen = 0
    for i, line in enumerate(lines):
        if "Compiling entry function" in line and any(kn in line for kn in XYZ_KERNELS):
            seen += 1
            block = "\n".join(lines[i:i + 4])
            mt = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", block)
            assert mt and mt.group(1) == "0" and mt.group(2) == "0", block
            fr = re.search(r"(\d+) bytes stack frame", block)
            assert fr and fr.group(1) == "0", block
    assert seen == 4, seen
