"""SpiderCNN training without a GPU: get_model_training's refusals, and the code shape of the training backward's kernels (no float
atomics, so a step is bit-reproducible, and no local-memory spills)."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest
import torch

from scanobjectnn_b200 import spidercnn_cls_xyz as M

KERNELS = ("spider_bwd_data_kernel", "spider_taylor_grad_kernel", "spider_taylor_grad_final_kernel", "spider_gn_bwd_kernel",
           "spider_gn_param_final_kernel", "train_gemm_kernelILi128ELi64ELb0ELb1ENS_7SpiderA")


def test_get_model_training_refuses_what_it_cannot_run():
    p = M.init_params(device="cpu")
    with pytest.raises(RuntimeError, match="CUDA"):
        M.get_model_training(torch.zeros((1, 32, 3)), params=p)
    with pytest.raises(NotImplementedError):
        M.get_model_training(torch.zeros((1, 32, 3), requires_grad=True), params=p)
    with pytest.raises(ValueError, match="num_class"):
        M.get_model_training(torch.zeros((1, 32, 3)), num_class=40, params=p)


def test_inference_get_model_points_at_get_model_training():
    with pytest.raises(NotImplementedError, match="get_model_training"):
        M.get_model(torch.zeros((1, 32, 3)), True, params=M.init_params(device="cpu"))


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_backward_kernels_have_no_float_atomics():
    from scanobjectnn_b200.build import build_library
    lib = build_library()
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if any(k in m.group(1) for k in KERNELS) else None
            if name:
                funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    assert all(any(k in f for f in funcs) for k in KERNELS), sorted(funcs)
    for f, lines in funcs.items():
        bad = [ln for ln in lines if re.search(r"\b(RED|ATOM|ATOMG|ATOMS)\b", ln)]
        assert not bad, (f, bad[:3])


def test_backward_kernels_do_not_spill():
    from scanobjectnn_b200.build import CSRC, NVCC_FLAGS, _nvcc
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([_nvcc(), *NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(CSRC, "spider.cu"), "-o", os.path.join(d, "s.o")],
                           capture_output=True, text=True, check=True)
    seen, name = set(), None
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1) if any(k in m.group(1) for k in KERNELS) else None
            continue
        if name is not None and "stack frame" in line:
            seen.add(name)
            assert re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", line), (name, line)
            name = None
    assert all(any(k in f for f in seen) for k in KERNELS), sorted(seen)
