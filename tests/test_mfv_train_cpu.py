"""3DmFV-Net training without a GPU: get_model_training's refusals, the training C entries' argument checks, the code shape of the
backward's kernels (no float atomics, so a step is bit-reproducible; no stack frame or spills), and the GPU tests' float64
restatement with batch norm frozen against the independent transcription oracle/mfv_oracle.py."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from oracle import mfv_oracle as mo
from scanobjectnn_b200 import mfv_net_cls as M
from scanobjectnn_b200.synthetic import make_clouds

from .restate import params_as
from .test_mfv_train_gpu import mfv_training

KERNELS = ("mfv_grad_finish_kernel", "mfv_bn_relu_kernel", "mfv_bn_dy_kernel", "mfv_maxpool_win_kernel", "mfv_maxpool_bwd_kernel",
           "mfv_avgpool_bwd_kernel", "train_gemm_kernelILi128ELi64ELb0ELb1ENS_8MfvConvA", "train_gemm_kernelILi128ELi64ELb1ELb0ENS_8MfvGradA")


def test_get_model_training_refuses_what_it_cannot_run():
    p = M.init_params(device="cpu")
    w, mu, s = M.get_3d_grid_gmm()
    with pytest.raises(RuntimeError, match="CUDA"):
        M.get_model_training(torch.zeros((1, 32, 3)), w, mu, s, params=p)
    with pytest.raises(NotImplementedError):
        M.get_model_training(torch.zeros((1, 32, 3), requires_grad=True), w, mu, s, params=p)
    with pytest.raises(NotImplementedError):
        M.get_model_training(torch.zeros((1, 32, 3)), w, mu, s, params=p, add_noise=True)
    with pytest.raises(ValueError, match="num_classes"):
        M.get_model_training(torch.zeros((1, 32, 3)), w, mu, s, num_classes=40, params=p)
    with pytest.raises(ValueError, match="cube"):
        M.get_model_training(torch.zeros((1, 32, 3)), w[:100], mu[:100], s[:100], params=p)


def test_inference_get_model_points_at_get_model_training():
    w, mu, s = M.get_3d_grid_gmm()
    with pytest.raises(NotImplementedError, match="get_model_training"):
        M.get_model(torch.zeros((1, 32, 3)), w, mu, s, True, params=M.init_params(device="cpu"))


def test_training_entries_reject_bad_arguments_without_a_gpu():
    from scanobjectnn_b200 import _lib
    lib = _lib.load()
    null = C.c_void_p(0)
    bw = lambda b, r, k, c, co, ldx: lib.psa_conv3d_bwd_weight(b, r, k, c, co, null, ldx, null, null, null, 0, null)   # noqa: E731
    bd = lambda b, r, k, c, co, ld: lib.psa_conv3d_bwd_data(b, r, k, c, co, null, null, null, ld, 0, null, 0, null)      # noqa: E731
    for f in (bw, bd):
        assert f(1, 5, 2, 64, 32, 64) == -1                                                 # k not in {1, 3, 5}
        assert f(1, 5, 3, 64, 32, 32) == -1                                                 # stride below the width
        assert f(1, 5, 3, 64, 32, 64) == -1                                                 # null buffers
        assert b"null buffer" in lib.psa_last_error()
        assert f(0, 5, 3, 64, 32, 64) == 0                                                  # zero batch: a no-op
        assert f(-1, 5, 3, 64, 32, 64) == -1
    assert lib.psa_conv3d_bwd_workspace_bytes(1, 5, 2, 64, 32) == 0
    assert lib.psa_conv3d_bwd_workspace_bytes(64, 5, 5, 256, 128) > 0
    assert lib.psa_mfv_bn_relu(10, 8, null, null, null, null, 4, null) == -1               # ldo below the width
    assert lib.psa_mfv_bn_relu(10, 8, null, null, null, null, 8, null) == -1
    assert lib.psa_mfv_bn_relu(0, 8, null, null, null, null, 8, null) == 0
    g = _lib.PsaGradIn(ld_dh=8, pool_k=1, C=8)
    assert lib.psa_mfv_bn_dy(10, 8, C.byref(g), null, null) == -1
    assert lib.psa_mfv_bn_dy(0, 8, C.byref(g), null, null) == 0
    assert lib.psa_pool3d_max_train(1, 5, 8, null, null, null, null) == -1
    assert lib.psa_pool3d_max_train(0, 5, 8, null, null, null, null) == 0
    assert lib.psa_pool3d_bwd(1, 5, 8, 2, null, null, null, null) == -1                     # kind not 0 / 1
    assert lib.psa_pool3d_bwd(1, 5, 8, 1, null, null, null, null) == -1
    assert lib.psa_pool3d_bwd(0, 5, 8, 1, null, null, null, null) == 0


def test_mac_counts_skip_the_out_of_grid_taps():
    from scanobjectnn_b200 import ops
    # a 1^3 conv has one tap, inside the grid for every row: nothing to skip
    assert ops.conv3d_bwd_macs(64, 5, 1, 384, 256) == (64 * 125 * 384 * 256,) * 3
    # inception3_conv3 at train.py's batch: in-grid MACs are 80 / 199 of the dense product, the issued ones close to them
    iw, idd, ig = ops.conv3d_bwd_macs(64, 5, 5, 256, 128)
    dense = 64 * 125 * 125 * 256 * 128
    assert ig == 64 * (3 + 4 + 5 + 4 + 3) ** 3 * 256 * 128
    assert ig <= iw < 1.05 * ig and ig <= idd < 1.5 * ig and idd < 0.6 * dense


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


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="nvcc not found")
def test_backward_kernels_do_not_spill():
    from scanobjectnn_b200.build import CSRC, NVCC_FLAGS, _nvcc
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([_nvcc(), *NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(CSRC, "mfv_train.cu"), "-o", os.path.join(d, "m.o")],
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


def test_restatement_with_frozen_batch_norm_matches_the_oracle():
    """the GPU tests' float64 restatement, batch norm on the moving averages, against oracle/mfv_oracle.py at B=2, N=256"""
    p = M.init_params(seed=3, device="cpu", randomize_bn=True)
    pts = make_clouds("ball", 2, 256, seed=33)
    w, mu, s = M.get_3d_grid_gmm()
    fv = mo.fisher_vector(pts, w, mu, s)
    want, _ = mo.forward_from_fv(fv, p)
    got = mfv_training(torch.from_numpy(fv), params_as(p, torch.float64), frozen=True)
    assert float(np.abs(got.numpy() - want.numpy()).max()) < 1e-10 * max(1.0, float(want.abs().max()))
