"""SASS shape of tc_sa_kernel's last layer (cuobjdump, no GPU needed).

In the 128-wide levels (PointNet++ SA2) a warpgroup issues the next 64-channel chunk of the last layer before the epilogue of
the current one, so it waits with one group still pending (`wgmma.wait_group 1` = `WARPGROUP.DEPBAR.LE gsb0, 0x1`) instead of
draining the tensor pipe after every chunk."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "scanobjectnn_b200", "libpsa.so")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")

SA2 = "_ZN3psa12tc_sa_kernelILi2ELi128ELi2ELi128EEEvNS_6TcArgsE"


def _sass(name):
    from scanobjectnn_b200.build import build_library
    build_library()
    out = subprocess.run(["cuobjdump", "-sass", "-fun", name, LIB], capture_output=True, text=True, check=True).stdout
    assert "HGMMA" in out, f"{name} not found in {LIB}"
    return out


def test_sa2_last_layer_keeps_one_wgmma_group_in_flight():
    text = _sass(SA2)
    waits = re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, (0x[0-9a-f]+)", text)
    assert "0x1" in waits, f"every wgmma wait drains the pipe: {sorted(set(waits))}"
