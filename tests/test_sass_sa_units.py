"""SASS code shape of tc_sa_kernel's tile loop (cuobjdump, no GPU needed).

The two warpgroups of a CTA work on their own tiles and synchronise on named barriers (one per warpgroup), so that one's
gathers and epilogues overlap the other's wgmma.  A CTA-wide __syncthreads (barrier 0) only remains in the set-up, before
the tile loop: one more would put the warpgroups back in lockstep."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "scanobjectnn_b200", "libpsa.so")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")


@pytest.fixture(scope="module")
def sa_kernels():
    from scanobjectnn_b200.build import build_library
    build_library()
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if "tc_sa_kernel" in m.group(1) else None
            if name:
                funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    assert len(funcs) == 12, sorted(funcs)          # NP in {2, 3} x six level shapes
    return funcs


def test_tc_sa_kernel_syncs_its_warpgroups_on_named_barriers(sa_kernels):
    for name, lines in sa_kernels.items():
        bars = [l for l in lines if re.search(r"\bBAR\.SYNC(\.\w+)*\b", l)]
        cta_wide = [l for l in bars if re.search(r"BAR\.SYNC(\.\w+)* 0x0\s*;", l)]
        named = [l for l in bars if re.search(r"BAR\.SYNC(\.\w+)* R\d+", l)]
        assert len(cta_wide) <= 1, f"{name}: {len(cta_wide)} CTA-wide barriers -- the warpgroups run in lockstep again"
        assert len(named) >= 3, f"{name}: {len(named)} named barriers (tile claim + two per pooled chunk expected)"


def test_sa1_shape_fits_two_ctas_per_sm(sa_kernels):
    """The 64-64-128 level (PointNet++ SA1) keeps <= 128 registers, so two 256-thread CTAs share an SM."""
    lines = sa_kernels["_ZN3psa12tc_sa_kernelILi2ELi64ELi2ELi64EEEvNS_6TcArgsE"]
    regs = [int(r) for l in lines for r in re.findall(r"\bR(\d+)\b", l)]
    assert max(regs) < 128, f"R{max(regs)} in use: one CTA per SM"
