"""SASS-level regression checks on the built library (cuobjdump, no GPU needed).

The hot kernels really contain the Hopper instructions they are written for (HGMMA = wgmma, bulk copies, mbarrier waits),
i.e. nothing fell back to a generic path, and the index kernels keep their code shape."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "scanobjectnn_b200", "libpsa.so")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")


@pytest.fixture(scope="module")
def sass():
    from scanobjectnn_b200.build import build_library
    build_library()
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    return funcs


def _count(lines, mnemonic):
    return sum(1 for l in lines if re.search(r"\b" + mnemonic + r"\b", l))


def _kernels(sass, pattern):
    ks = {k: v for k, v in sass.items() if pattern in k}
    assert ks, f"no kernel matching {pattern}"
    return ks


def test_default_kernels_contain_the_hopper_instructions(sass):
    for pattern, needed in {"tc_sa_kernel": ["HGMMA", "UBLKCP", "SYNCS"],
                            "tc_dense_kernel": ["HGMMA", "UBLKCP", "SYNCS"],
                            "knn_tc_kernel": ["HGMMA", "UBLKCP", "SYNCS"]}.items():
        ks = _kernels(sass, pattern)
        for name, lines in ks.items():
            text = "\n".join(lines)
            for mn in needed:
                assert re.search(r"\b" + mn, text), f"{name}: no {mn} in SASS"
            assert _count(lines, r"HGMMA(\.\w+)*") >= 12, name
    assert len(_kernels(sass, "tc_sa_kernel")) >= 2 and len(_kernels(sass, "tc_dense_kernel")) >= 2     # fp16x2 and bf16x3 instantiations


def test_index_kernels_use_redux(sass):
    fps = "\n".join(l for k, v in _kernels(sass, "fps_kernel").items() for l in v)
    assert re.search(r"\bREDUX\b|\bCREDUX\b", fps), "FPS lost its warp REDUX arg-max"


def test_streaming_f1_kernel_keeps_its_code_shape(sass):
    """sa_conv1_stream_kernel (DESIGN.md 3.5): the search is unrolled over the thread's point pairs with funnel shifts collecting the
    sign masks (no per-word ballots: VOTE only in the extraction's bookkeeping), the warpgroups re-partition their registers with
    setmaxnreg, the output leaves in 128-bit evict-first streaming stores, and the 128-register search stage does not spill beyond a
    few words."""
    ks = _kernels(sass, "sa_conv1_stream_kernel")
    assert len(ks) == 12, sorted(ks)                  # NV in {2, 4} x HAS_U x PPTP in {8, 16, 32}
    for name, lines in ks.items():
        text = "\n".join(lines)
        pptp = int(re.search(r"ELi(\d+)EEEv", name).group(1))
        pairs = pptp // 2                             # point pairs per thread = unrolled distance tests
        assert _count(lines, "FMUL") >= 2 * pairs and _count(lines, "FFMA") >= 4 * pairs and _count(lines, "FADD") >= 8 * pairs, name
        assert _count(lines, r"SHF(\.\w+)*") >= 2 * pairs, f"{name}: the sign-mask funnel shifts are gone"
        assert _count(lines, r"VOTE(\.\w+)*") <= 8, f"{name}: ballots are back in the search"
        assert _count(lines, "USETMAXREG") >= 3, f"{name}: no setmaxnreg"
        assert re.search(r"STG\.E\.EF\.128", text), f"{name}: output no longer leaves in 128-bit evict-first stores"
        assert _count(lines, r"STL(\.\w+)*") <= 40 and _count(lines, r"LDL(\.\w+)*") <= 40, f"{name}: register spills"   # scalar f32 pairs on sm_90: more live registers
        assert not re.search(r"\bRED\b|\bATOMG\b.*\.F32", text), f"{name}: float atomics in the statistics"


def test_wgmma_sequences_are_not_serialized(sass):
    """Every HGMMA kernel issues its wgmma in straight-line groups: one WARPGROUP.ARRIVE per group, not one per HGMMA.  (ptxas
    inserts an arrive before each wgmma -- and serialises them, warning C7520 -- when the issue sits on a runtime-predicated path.)"""
    for pattern in ("tc_sa_kernel", "tc_dense_kernel", "knn_tc_kernel"):
        for name, lines in _kernels(sass, pattern).items():
            hgmma, arrive = _count(lines, r"HGMMA(\.\w+)*"), _count(lines, r"WARPGROUP\.ARRIVE")
            assert arrive >= 1 and 4 * arrive <= hgmma, f"{name}: {arrive} WARPGROUP.ARRIVE for {hgmma} HGMMA -- the wgmma are serialized"
