"""SASS code shape of the shared ring GEMM (csrc/ring_gemm.cuh) in all twelve instantiations: tc_spider_kernel, tc_conv3d_kernel and
tc_pcnn_dense_kernel, each for NP in {2, 3} x NC in {1, 2} (cuobjdump, no GPU needed).

Each one stages blocks by TMA bulk copies and cp.async on mbarriers, issues its wgmma in straight-line groups, and hands the producers'
registers to the consumers by setmaxnreg: 40 and 232 from 168 at launch.  The hand-off needs exactly 168, since
128 * 40 + 256 * 232 = 384 * 168; with any other count setmaxnreg.inc waits for registers nobody releases."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "scanobjectnn_b200", "libpsa.so")
RING = ("tc_spider_kernel", "tc_conv3d_kernel", "tc_pcnn_dense_kernel")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")


@pytest.fixture(scope="module")
def cuobjdump():
    from scanobjectnn_b200.build import build_library
    build_library()
    return lambda flag: subprocess.run(["cuobjdump", flag, LIB], capture_output=True, text=True, check=True).stdout


def test_ring_kernels_code_shape(cuobjdump):
    funcs, name = {}, None
    for line in cuobjdump("-sass").splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if any(k in m.group(1) for k in RING) else None
            if name:
                funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    assert len(funcs) == 12, sorted(funcs)           # 3 ops x NP in {2, 3} x NC in {1, 2}
    for name, lines in funcs.items():
        text = "\n".join(lines)
        for mn in ("HGMMA", "UBLKCP", "SYNCS", "LDGSTS"):
            assert re.search(r"\b" + mn, text), f"{name}: no {mn}"
        hgmma = sum(1 for l in lines if re.search(r"\bHGMMA(\.\w+)*", l))
        arrive = sum(1 for l in lines if "WARPGROUP.ARRIVE" in l)
        assert arrive >= 1 and 4 * arrive <= hgmma, f"{name}: {arrive} WARPGROUP.ARRIVE for {hgmma} HGMMA -- serialized"
        assert sum(1 for l in lines if "USETMAXREG" in l) >= 2, f"{name}: no setmaxnreg"
        assert not any(re.search(r"\b(STL|LDL)\b", l) for l in lines), f"{name}: register spills"


def test_ring_kernels_launch_with_168_registers_and_no_stack(cuobjdump):
    """the registers ptxas allotted (cuobjdump -res-usage), and no stack frame"""
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:\d+ STACK:\d+)", cuobjdump("-res-usage")))
    ring = {k: v for k, v in usage.items() if any(n in k for n in RING)}
    assert len(ring) == 12, sorted(ring)
    for name, res in ring.items():
        assert res.startswith("REG:168 STACK:0"), f"{name}: {res}"
