"""SASS code shape of tc_dense_kernel (cuobjdump, no GPU needed).

The kernel is persistent and warp-specialised: a producer warp streams x and weight blocks through an mbarrier ring, and the
two consumer warpgroups never wait for each other inside the K loop.  A CTA-wide __syncthreads (barrier 0) only remains in
the set-up, before the tile loop; the epilogue's cross-warp pooling and statistics use a named barrier of the consumers."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "scanobjectnn_b200", "libpsa.so")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")


@pytest.fixture(scope="module")
def dense_kernels():
    from scanobjectnn_b200.build import build_library
    build_library()
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if "tc_dense_kernel" in m.group(1) else None
            if name:
                funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    assert len(funcs) == 4, sorted(funcs)           # NP in {2, 3} x NC in {1, 2}
    return funcs


def test_tc_dense_kernel_has_no_cta_wide_barrier_in_its_tile_loop(dense_kernels):
    for name, lines in dense_kernels.items():
        bars = [l for l in lines if re.search(r"\bBAR\.SYNC(\.\w+)*\b", l)]
        cta_wide = [l for l in bars if re.search(r"BAR\.SYNC(\.\w+)* 0x0\s*;", l)]
        assert len(cta_wide) <= 1, f"{name}: {len(cta_wide)} CTA-wide barriers -- the consumers wait for each other again"
        assert len(bars) > len(cta_wide), f"{name}: no named barrier for the epilogue"


def test_tc_dense_kernel_is_warp_specialised(dense_kernels):
    """The producer warpgroup gives its registers to the consumers (setmaxnreg) and nothing spills."""
    for name, lines in dense_kernels.items():
        assert sum(1 for l in lines if "USETMAXREG" in l) >= 2, f"{name}: no setmaxnreg"
        assert not any(re.search(r"\b(STL|LDL)\b", l) for l in lines), f"{name}: register spills"
