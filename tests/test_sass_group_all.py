"""SASS code shape of tc_group_all_kernel (cuobjdump and ptxas, no GPU needed).

The group-all level's cluster kernel keeps tc_dense_kernel's structure: a producer warp streams weight blocks with bulk copies
through an mbarrier ring, the producer warpgroup gives its registers to the two consumer warpgroups, nothing spills, and the
wgmma of a K block issue as one straight-line group."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "scanobjectnn_b200", "libpsa.so")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("nvcc") is None, reason="CUDA tools not on PATH")


@pytest.fixture(scope="module")
def group_all_kernels():
    from scanobjectnn_b200.build import build_library
    build_library()
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if "tc_group_all_kernel" in m.group(1) else None
            if name:
                funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    assert len(funcs) == 3, sorted(funcs)           # (layer-0, layer-1 slice chunks) in {(1, 1), (1, 2), (2, 1)}
    return funcs


def _count(lines, pattern):
    return sum(1 for l in lines if re.search(pattern, l))


def test_group_all_kernel_is_warp_specialised_tma_and_wgmma(group_all_kernels):
    for name, lines in group_all_kernels.items():
        assert _count(lines, r"\bHGMMA\b") > 0, f"{name}: no wgmma"
        assert _count(lines, r"\bUBLKCP\b") > 0, f"{name}: no bulk copies"
        assert _count(lines, r"\bSYNCS\b") > 0, f"{name}: no mbarrier operations"
        assert _count(lines, r"USETMAXREG") >= 2, f"{name}: no setmaxnreg"
        assert _count(lines, r"\b(STL|LDL)\b") == 0, f"{name}: register spills"


def test_group_all_kernel_issues_wgmma_in_groups(group_all_kernels):
    for name, lines in group_all_kernels.items():
        hgmma, arrive = _count(lines, r"\bHGMMA\b"), _count(lines, r"WARPGROUP\.ARRIVE")
        assert arrive > 0 and hgmma >= 4 * arrive, f"{name}: {hgmma} HGMMA for {arrive} WARPGROUP.ARRIVE"


def test_ptxas_does_not_serialise_wgmma(tmp_path):
    """C7514 / C7518 / C7520: ptxas serialised wgmma (register use across the async boundary, a predicated issue, ...)"""
    from scanobjectnn_b200 import build
    src = os.path.join(build.CSRC, "tc_mlp.cu")
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-I", os.path.join(ROOT, "include"), "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "tc_mlp.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    assert "tc_group_all_kernel" in log
    bad = [l for l in log.splitlines() if re.search(r"C75(14|18|20)", l)]
    assert not bad, "\n".join(bad)
