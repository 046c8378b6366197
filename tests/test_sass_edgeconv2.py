"""SASS code shape of the two-layer training EdgeConv kernels (cuobjdump, no GPU needed): the per-edge products run on wgmma issued
in straight-line groups, nothing spills, and no reduction uses float atomics (every sum is added in a fixed order)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "scanobjectnn_b200", "libpsa.so")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")


@pytest.fixture(scope="module")
def edge2_kernels():
    from scanobjectnn_b200.build import build_library
    build_library()
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if "edge2_" in m.group(1) else None
            if name:
                funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    return funcs


def test_edgeconv2_products_run_on_wgmma_in_straight_line_groups(edge2_kernels):
    mma = {k: v for k, v in edge2_kernels.items() if "edge2_train_kernel" in k}
    assert len(mma) == 4, sorted(mma)              # statistics, pooling, dW2, dh1
    for name, lines in mma.items():
        hgmma = sum(1 for l in lines if "HGMMA" in l)
        arrive = sum(1 for l in lines if "WARPGROUP.ARRIVE" in l)
        assert hgmma > 0, f"{name}: no HGMMA"
        assert 4 * arrive <= hgmma, f"{name}: {arrive} WARPGROUP.ARRIVE for {hgmma} HGMMA -- the wgmma sequence was serialised"


def test_edgeconv2_kernels_do_not_spill_or_use_float_atomics(edge2_kernels):
    assert edge2_kernels
    for name, lines in edge2_kernels.items():
        assert not any(re.search(r"\b(STL|LDL)\b", l) for l in lines), f"{name}: register spills"
        assert not any(re.search(r"\bRED\b|\bRED\.|ATOMG\S*F32", l) for l in lines), f"{name}: float atomics"
