"""SASS code shape of the shared ring GEMM (csrc/ring_gemm.cuh) in all sixteen instantiations: tc_dense_kernel, tc_spider_kernel,
tc_conv3d_kernel and tc_pcnn_dense_kernel, each for NP in {2, 3} x NC in {1, 2} (cuobjdump, no GPU needed).

Each one stages blocks by TMA bulk copies and cp.async on mbarriers, issues its wgmma in straight-line groups, and hands the producers'
registers to the consumers by setmaxnreg: 40 and 232 from 168 at launch.  The hand-off needs exactly 168, since
128 * 40 + 256 * 232 = 384 * 168; with any other count setmaxnreg.inc waits for registers nobody releases.

The consumer warpgroups never wait for each other inside the K loop: a CTA-wide __syncthreads (barrier 0) only remains in the set-up,
and the dense op's cross-warp pooling and statistics use a named barrier of the consumers."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "scanobjectnn_b200", "libpsa.so")
RING = ("tc_dense_kernel", "tc_spider_kernel", "tc_conv3d_kernel", "tc_pcnn_dense_kernel")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")


@pytest.fixture(scope="module")
def cuobjdump():
    from scanobjectnn_b200.build import build_library
    build_library()
    return lambda flag: subprocess.run(["cuobjdump", flag, LIB], capture_output=True, text=True, check=True).stdout


@pytest.fixture(scope="module")
def ring_sass(cuobjdump):
    funcs, name = {}, None
    for line in cuobjdump("-sass").splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if any(k in m.group(1) for k in RING) else None
            if name:
                funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    assert len(funcs) == 16, sorted(funcs)           # 4 ops x NP in {2, 3} x NC in {1, 2}
    return funcs


def test_ring_kernels_code_shape(ring_sass):
    for name, lines in ring_sass.items():
        text = "\n".join(lines)
        for mn in ("HGMMA", "UBLKCP", "SYNCS", "LDGSTS"):
            assert re.search(r"\b" + mn, text), f"{name}: no {mn}"
        hgmma = sum(1 for l in lines if re.search(r"\bHGMMA(\.\w+)*", l))
        arrive = sum(1 for l in lines if "WARPGROUP.ARRIVE" in l)
        assert arrive >= 1 and 4 * arrive <= hgmma, f"{name}: {arrive} WARPGROUP.ARRIVE for {hgmma} HGMMA -- serialized"
        assert sum(1 for l in lines if "USETMAXREG" in l) >= 2, f"{name}: no setmaxnreg"
        assert not any(re.search(r"\b(STL|LDL)\b", l) for l in lines), f"{name}: register spills"


def test_dense_ring_kernel_has_no_cta_wide_barrier_in_its_unit_loop(ring_sass):
    dense = {k: v for k, v in ring_sass.items() if "tc_dense_kernel" in k}
    assert len(dense) == 4, sorted(dense)
    for name, lines in dense.items():
        bars = [l for l in lines if re.search(r"\bBAR\.SYNC(\.\w+)*\b", l)]
        cta_wide = [l for l in bars if re.search(r"BAR\.SYNC(\.\w+)* 0x0\s*;", l)]
        assert len(cta_wide) <= 1, f"{name}: {len(cta_wide)} CTA-wide barriers -- the consumers wait for each other again"
        assert len(bars) > len(cta_wide), f"{name}: no named barrier for the epilogue"


def test_dense_ring_kernel_is_warp_specialised(ring_sass):
    """The dense op's producers (staging, unit claims) give their registers to the consumers: setmaxnreg down to 40 and up to 232,
    and nothing spills on either side of the hand-off."""
    dense = {k: v for k, v in ring_sass.items() if "tc_dense_kernel" in k}
    assert len(dense) == 4, sorted(dense)
    for name, lines in dense.items():
        assert any(re.search(r"USETMAXREG\.DEALLOC(\.\w+)* 0x28\b", l) for l in lines), f"{name}: producers keep more than 40 registers"
        assert any(re.search(r"USETMAXREG\.TRY_ALLOC(\.\w+)* \w+, 0xe8\b", l) for l in lines), f"{name}: consumers do not take 232 registers"
        assert not any(re.search(r"\b(STL|LDL)\b", l) for l in lines), f"{name}: register spills"


def test_ring_kernels_launch_with_168_registers_and_no_stack(cuobjdump):
    """the registers ptxas allotted (cuobjdump -res-usage), and no stack frame"""
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:\d+ STACK:\d+)", cuobjdump("-res-usage")))
    ring = {k: v for k, v in usage.items() if any(n in k for n in RING)}
    assert len(ring) == 16, sorted(ring)
    for name, res in ring.items():
        assert res.startswith("REG:168 STACK:0"), f"{name}: {res}"
