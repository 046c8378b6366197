"""3DmFV-Net without a GPU: the grid GMM against the reference's own function (golden data), the reference's variable names and
shapes and a TF checkpoint round trip, the float64 restatement (oracle/mfv_oracle.py) against a literal tiled transcription of
get_3dmfv and its pools against loops with TF's SAME padding, the refusals of the model and the C ABI's argument checks."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import mfv_oracle as mo
from scanobjectnn_b200 import checkpoint as ck
from scanobjectnn_b200 import mfv_net_cls as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_3dmfv_grid_gmm.npz")
LIB = os.path.join(ROOT, "scanobjectnn_b200", "libpsa.so")


@pytest.mark.parametrize("r", [3, 5, 8])
def test_grid_gmm_matches_the_reference(r):
    z = np.load(GOLDEN)
    w, mu, sigma = M.get_3d_grid_gmm((r, r, r), 0.04)
    assert np.array_equal(w, z[f"w{r}"].astype(np.float32))
    assert np.array_equal(mu, z[f"mu{r}"].astype(np.float32))
    assert np.array_equal(sigma, np.sqrt(z[f"cov{r}"]).astype(np.float32))        # train.py feeds sqrt(covariances_)
    g = np.arange(r ** 3)                                                          # Gaussian g at cell (g // r^2, g // r % r, g % r)
    step = 2.0 / r
    np.testing.assert_allclose(mu, np.stack([g // r ** 2, g // r % r, g % r], 1) * step - 1 + step / 2, atol=1e-6)


def _reference_shapes(num_classes=15):
    """3dmfv_net_cls.py:29-102 with tf_util.conv3d's variables (weights (k,k,k,cin,cout), biases, bn/*) and fully_connected's"""
    want, cin = {}, 20
    for l, n in enumerate((64, 128, 256, 256, 512), start=1):
        for j, (k, a, b) in enumerate([(1, cin, n), (3, n, n // 2), (5, n, n // 2), (1, cin, n)], start=1):
            s = f"inception{l}_conv{j}"
            want[f"{s}/weights"] = (k, k, k, a, b)
            want[f"{s}/biases"] = (b,)
            for v in ("beta", "gamma", "moving_mean", "moving_variance"):
                want[f"{s}/bn/{v}"] = (b,)
        cin = 3 * n
    for scope, (a, b) in {"fc1": (2 * 2 * 2 * 1536, 1024), "fc2": (1024, 256), "fc3": (256, 128)}.items():
        want[f"{scope}/weights"] = (a, b)
        want[f"{scope}/biases"] = (b,)
        for v in ("beta", "gamma", "moving_mean", "moving_variance"):
            want[f"{scope}/bn/{v}"] = (b,)
    want["fc4/weights"] = (128, num_classes)
    want["fc4/biases"] = (num_classes,)
    return want


def test_init_params_has_the_reference_variables():
    p = M.init_params(device="cpu")
    assert {k: tuple(v.shape) for k, v in p.items()} == _reference_shapes()
    # Xavier limits of TF's 5-D rule: fan_in k^3 cin, fan_out k^3 cout
    assert float(p["inception3_conv3/weights"].abs().max()) <= np.sqrt(6.0 / (125 * 256 + 125 * 128))
    assert float(p["inception3_conv3/weights"].abs().max()) > 0.9 * np.sqrt(6.0 / (125 * 256 + 125 * 128))
    assert float(p["inception1_conv1/weights"].abs().max()) <= np.sqrt(6.0 / (20 + 64))
    assert set(M.init_params(num_classes=40, device="cpu")["fc4/biases"].shape) == {40}


def test_store_survives_a_tf_checkpoint_round_trip(tmp_path):
    p = M.init_params(seed=2, device="cpu", randomize_bn=True)
    src = {k: v.numpy().copy() for k, v in p.items()}
    prefix = str(tmp_path / "model.ckpt")
    ck.write_tf_checkpoint(prefix, src)
    q = M.init_params(seed=7, device="cpu")
    assert ck.restore(q, prefix) == []
    for k in p:
        assert q[k].shape == p[k].shape and np.array_equal(q[k].numpy(), src[k]), k


def test_refusals():
    p = M.init_params(device="cpu")
    w, mu, s = M.get_3d_grid_gmm()
    with pytest.raises(NotImplementedError):
        M.get_model(torch.zeros((1, 32, 3)), w, mu, s, True, params=p)
    with pytest.raises(NotImplementedError):
        M.get_model(torch.zeros((1, 32, 3), requires_grad=True), w, mu, s, False, params=p)
    with pytest.raises(NotImplementedError):
        M.get_model(torch.zeros((1, 32, 3)), w, mu, s, False, add_noise=True, params=p)
    with pytest.raises(ValueError):
        M.get_model(torch.zeros((1, 32, 3)), w, mu, s, False, num_classes=40, params=p)


def _tiled_fisher_vector(points, w, mu, sigma):
    """tf_util.get_3dmfv (flatten=False) transcribed with the reference's own tiles: batch_sig, batch_mu, batch_w, batch_points
    (B,N,G,D), the density of MultivariateNormalDiag evaluated per tiled entry, then the derivatives and normalisations"""
    B, N, D = points.shape
    G = mu.shape[0]
    batch_sig = np.tile(sigma[None, None], [B, N, 1, 1])
    batch_mu = np.tile(mu[None, None], [B, N, 1, 1])
    batch_w = np.tile(w[None, None], [B, N, 1])
    batch_points = np.tile(points[:, :, None, :], [1, 1, G, 1])
    w_per_batch_per_d = np.tile(w[None, :, None], [B, 1, 3 * D])
    p = np.zeros((B, N, G))
    for b in range(B):
        for i in range(N):
            for g in range(G):
                dens = 1.0
                for d in range(D):
                    s = batch_sig[b, i, g, d]
                    dens *= np.exp(-0.5 * ((batch_points[b, i, g, d] - batch_mu[b, i, g, d]) / s) ** 2) / (np.sqrt(2 * np.pi) * s)
                p[b, i, g] = dens
    w_p = p * batch_w
    Q = w_p / np.tile(w_p.sum(-1)[..., None], [1, 1, G])
    Q_per_d = np.tile(Q[..., None], [1, 1, 1, D])
    d_pi_all = ((Q - batch_w) / (np.sqrt(batch_w) * N))[..., None]
    d_pi = np.concatenate([d_pi_all.max(1), d_pi_all.sum(1)], axis=2)
    d_mu_all = Q_per_d * (batch_points - batch_mu) / batch_sig
    d_mu = (1 / (N * np.sqrt(w_per_batch_per_d))) * np.concatenate([d_mu_all.max(1), d_mu_all.min(1), d_mu_all.sum(1)], axis=2)
    d_sig_all = Q_per_d * (((batch_points - batch_mu) / batch_sig) ** 2 - 1)
    d_sigma = (1 / (N * np.sqrt(2 * w_per_batch_per_d))) * np.concatenate([d_sig_all.max(1), d_sig_all.min(1), d_sig_all.sum(1)], axis=2)
    parts = []
    for v in (d_pi, d_mu, d_sigma):
        v = np.sign(v) * np.power(np.abs(v), 0.5)
        parts.append(v / np.sqrt(np.maximum(np.sum(v ** 2, axis=1, keepdims=True), 1e-12)))
    return np.concatenate(parts, axis=2)                                  # (B,G,20) = fv before its transpose to (B,20,G)


def test_oracle_fisher_vector_matches_the_tiled_transcription():
    from scanobjectnn_b200.synthetic import make_clouds
    pts = make_clouds("ball", 2, 64, seed=4).astype(np.float64)
    w, mu, sigma = (a.astype(np.float64) for a in M.get_3d_grid_gmm((3, 3, 3)))
    want = _tiled_fisher_vector(pts, w, mu, sigma)
    got = mo.fisher_vector(pts, w, mu, sigma)
    assert got.shape == (2, 27, 20)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)


def _tf_same_pads(r, k, s):
    out = -(-r // s)
    total = max((out - 1) * s + k - r, 0)
    return out, total // 2                                                 # TF: the smaller half before, the rest after


def _loop_pool(x, k, s, op):
    """tf.nn.{avg,max}_pool3d with SAME padding, by loops: pad cells are left out (avg divides by the in-grid count)"""
    b, c, r = x.shape[0], x.shape[1], x.shape[2]
    out_r, before = _tf_same_pads(r, k, s)
    out = np.zeros((b, c, out_r, out_r, out_r))
    for i in range(out_r):
        for j in range(out_r):
            for l in range(out_r):
                cells = [(i * s - before + a, j * s - before + bb, l * s - before + cc) for a in range(k) for bb in range(k) for cc in range(k)]
                cells = [t for t in cells if all(0 <= u < r for u in t)]
                vals = np.stack([x[:, :, a, bb, cc] for a, bb, cc in cells], -1)
                out[:, :, i, j, l] = vals.mean(-1) if op == "avg" else vals.max(-1)
    return out


@pytest.mark.parametrize("r", [5, 3])
def test_oracle_pools_are_tf_same(r):
    x = torch.randn((2, 4, r, r, r), generator=torch.Generator().manual_seed(r), dtype=torch.float64)
    np.testing.assert_allclose(mo.avg_pool3(x).numpy(), _loop_pool(x.numpy(), 3, 1, "avg"), rtol=0, atol=1e-15)
    assert np.array_equal(mo.max_pool2(x).numpy(), _loop_pool(x.numpy(), 2, 2, "max"))
    assert mo.max_pool2(x).shape[2] == (r + 1) // 2


def test_invalid_arguments_are_rejected_without_a_gpu():
    from scanobjectnn_b200 import _lib
    lib = _lib.load()
    null = C.c_void_p(0)
    assert lib.psa_fisher_vector(-1, 16, 27, *[null] * 5, null) == -1
    assert lib.psa_fisher_vector(1, 16, 0, *[null] * 5, null) == -1
    assert lib.psa_fisher_vector(1, 16, 27, *[null] * 5, null) == -1                       # null buffers
    assert lib.psa_fisher_vector(1, 100000, 512, *[null] * 5, null) == -2                  # beyond one block's shared memory
    assert lib.psa_fisher_vector(0, 16, 27, *[null] * 5, null) == 0
    conv = lambda b, r, k, c, co, ldx, ldo: lib.psa_conv3d_infer(b, r, k, c, co, null, ldx, null, null, null, 1, null, ldo, null, 0, null)
    assert conv(1, 5, 2, 64, 32, 64, 32) == -1                                              # k not in {1, 3, 5}
    assert conv(1, 5, 3, 64, 32, 32, 32) == -1                                              # ldx below c
    assert conv(1, 5, 3, 64, 32, 64, 16) == -1                                              # ldo below c_out
    assert conv(1, 5, 3, 64, 32, 64, 32) == -1                                              # null buffers
    assert b"null buffer" in lib.psa_last_error()
    assert conv(0, 5, 3, 64, 32, 64, 32) == 0
    assert lib.psa_conv3d_workspace_bytes(1, 5, 2, 64, 32) == 0
    assert lib.psa_conv3d_workspace_bytes(32, 5, 1, 20, 64) == 0                           # c = 20 runs on the FMA kernel
    assert lib.psa_conv3d_workspace_bytes(32, 3, 5, 512, 256) > 0
    assert lib.psa_pool3d(1, 5, 8, 2, null, null, null) == -1
    assert lib.psa_pool3d(1, 0, 8, 0, null, null, null) == -1


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_conv3d_kernel_code_shape():
    """tc_conv3d_kernel: wgmma, bulk copies and mbarriers in every instantiation, wgmma issued in straight-line groups, the
    producers' registers handed to the consumers; no local memory in any kernel of mfv.cu."""
    from scanobjectnn_b200.build import build_library
    build_library()
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    kernels = ("tc_conv3d_kernel", "conv3d_fma_kernel", "fisher_vector_kernel", "pool3d_", "conv3d_tapmask", "conv3d_finalize", "conv3d_pad")
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if any(k in m.group(1) for k in kernels) else None
            if name:
                funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    tc = {k: v for k, v in funcs.items() if "tc_conv3d_kernel" in k}
    assert len(tc) == 4, sorted(tc)                  # NP in {2, 3} x NC in {1, 2}
    assert len(funcs) == 11, sorted(funcs)
    for name, lines in tc.items():
        text = "\n".join(lines)
        for mn in ("HGMMA", "UBLKCP", "SYNCS", "LDGSTS"):
            assert re.search(r"\b" + mn, text), f"{name}: no {mn}"
        hgmma = sum(1 for l in lines if re.search(r"\bHGMMA(\.\w+)*", l))
        arrive = sum(1 for l in lines if "WARPGROUP.ARRIVE" in l)
        assert arrive >= 1 and 4 * arrive <= hgmma, f"{name}: {arrive} WARPGROUP.ARRIVE for {hgmma} HGMMA -- serialized"
        assert sum(1 for l in lines if "USETMAXREG" in l) >= 2, f"{name}: no setmaxnreg"
    for name, lines in funcs.items():
        assert not any(re.search(r"\b(STL|LDL)\b", l) for l in lines), f"{name}: local memory (spills)"


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not on PATH")
def test_ptxas_reports_no_spills_and_no_serialised_wgmma(tmp_path):
    from scanobjectnn_b200 import build
    src = os.path.join(build.CSRC, "mfv.cu")
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "mfv.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(frames) == 11 and all(f == ("0", "0", "0") for f in frames), frames
    assert not [l for l in log.splitlines() if re.search(r"C75(14|18|20)", l)]
