"""SpiderCNN without a GPU: the float64 restatement (oracle/spidercnn_oracle.py) against a plain-loop transcription of the
reference at a tiny size with the real channel widths, the reference's variable names and shapes and a TF checkpoint round trip,
the refusal of training mode and the C ABI's argument checks (the fused kernel's code shape: test_sass_ring.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import spidercnn_oracle as so
from scanobjectnn_b200 import checkpoint as ck
from scanobjectnn_b200 import spidercnn_cls_xyz as M

def _reference_shapes(num_class=15):
    want = {}
    cin = 3
    for l, cout in enumerate((32, 64, 128, 256), start=1):
        s = f"fanConv{l}/taylor"
        for m in ("x", "y", "z", "xyz", "xy", "yz", "xz", "xx", "yy", "zz", "xxy", "xyy", "xxz", "xzz", "yyz", "yzz", "xxx", "yyy", "zzz"):
            want[f"{s}/weight_{m}"] = (1, 1, 1, 5)
        want[f"{s}/biases"] = (1, 1, 1, 5)
        want[f"{s}/conv/weights"] = (1, 20, 5 * cin, cout)
        want[f"{s}/conv/biases"] = (cout,)
        want[f"{s}/conv/gn/gamma"] = (cout,)
        want[f"{s}/conv/gn/beta"] = (cout,)
        cin = cout
    for scope, (a, b) in {"fc1": (960, 1024), "fc2": (1024, 512)}.items():
        want[f"{scope}/weights"] = (a, b)
        want[f"{scope}/biases"] = (b,)
        for v in ("beta", "gamma", "moving_mean", "moving_variance"):
            want[f"{scope}/bn/{v}"] = (b,)
    want["fc3/weights"] = (512, num_class)
    want["fc3/biases"] = (num_class,)
    return want


def test_init_params_has_the_reference_variables():
    p = M.init_params(device="cpu")
    assert {k: tuple(v.shape) for k, v in p.items()} == _reference_shapes()
    # Xavier limits of TF's 4-D rule: Taylor vectors fan_in 1, fan_out 5; the conv fan_in 20*5*C_in, fan_out 20*C_out
    assert float(p["fanConv2/taylor/weight_x"].abs().max()) <= 1.0
    assert float(p["fanConv2/taylor/biases"].abs().max()) == 0.0
    assert float(p["fanConv4/taylor/conv/weights"].abs().max()) <= np.sqrt(6.0 / (20 * 5 * 128 + 20 * 256))


def test_store_survives_a_tf_checkpoint_round_trip(tmp_path):
    p = M.init_params(seed=2, device="cpu", randomize_bn=True)
    src = {k: v.numpy().copy() for k, v in p.items()}
    prefix = str(tmp_path / "model.ckpt")
    ck.write_tf_checkpoint(prefix, src)
    q = M.init_params(seed=7, device="cpu")
    assert ck.restore(q, prefix) == []
    for k in p:
        assert q[k].shape == p[k].shape and np.array_equal(q[k].numpy(), src[k]), k


def test_training_mode_is_refused():
    p = M.init_params(device="cpu")
    with pytest.raises(NotImplementedError):
        M.get_model(torch.zeros((1, 32, 3)), True, params=p)
    with pytest.raises(NotImplementedError):
        M.get_model(torch.zeros((1, 32, 3), requires_grad=True), False, params=p)


def _mono(name, d):
    """the monomial a variable name stands for: weight_xxy -> X^2 Y, biases -> 1 (parsed from the name, not from a table)"""
    if name == "biases":
        return 1.0
    out = 1.0
    for ch in name[len("weight_"):]:
        out *= d["xyz".index(ch)]
    return out


def _loop_forward(xyz, idx, p):
    """tf_util.spiderConv / group_norm_for_conv / topk_pool and the FC head, transcribed with loops over the indices"""
    b, n, k = idx.shape
    P = {key: v.double().numpy() for key, v in p.items()}
    names = [key.split("/")[-1] for key in P if key.startswith("fanConv1/taylor/") and "/conv/" not in key]
    feat = xyz.astype(np.float64)
    cat = []
    for l, cout in enumerate((32, 64, 128, 256), start=1):
        s = f"fanConv{l}/taylor"
        cin = feat.shape[2]
        T = P[f"{s}/biases"].shape[-1]
        W = P[f"{s}/conv/weights"]
        y = np.zeros((b, n, cout))
        for bi in range(b):
            for i in range(n):
                row = np.zeros(k * cin * T)
                for j in range(k):
                    nb = idx[bi, i, j]
                    d = xyz[bi, nb].astype(np.float64) - xyz[bi, i].astype(np.float64)
                    gt = np.zeros(T)
                    for nm in names:
                        gt += P[f"{s}/{nm}"].reshape(T) * _mono(nm, d)
                    for c in range(cin):
                        for t in range(T):
                            row[j * cin * T + c * T + t] = feat[bi, nb, c] * gt[t]      # channel c*T + t of slot j
                y[bi, i] = row @ W.reshape(k * cin * T, cout) + P[f"{s}/conv/biases"]
        G = min(16, cout)
        cpg = cout // G
        h = np.zeros_like(y)
        for bi in range(b):
            for g in range(G):
                chans = range(g * cpg, (g + 1) * cpg)                                     # contiguous groups
                vals = y[bi][:, g * cpg:(g + 1) * cpg]
                mean, var = vals.mean(), vals.var()
                for ch in chans:
                    h[bi, :, ch] = (y[bi, :, ch] - mean) / np.sqrt(var + 1e-6) * P[f"{s}/conv/gn/gamma"][ch] + P[f"{s}/conv/gn/beta"][ch]
        h = np.maximum(h, 0.0)
        cat.append(h)
        feat = h
    cat = np.concatenate(cat, axis=2)
    pooled = np.zeros((b, 2 * cat.shape[2]))
    for bi in range(b):
        for c in range(cat.shape[2]):
            top = sorted(cat[bi, :, c], reverse=True)[:2]
            for r in range(2):
                pooled[bi, c * 2 + r] = top[r]
    net = pooled
    for scope in ("fc1", "fc2"):
        z = net @ P[f"{scope}/weights"] + P[f"{scope}/biases"]
        z = (z - P[f"{scope}/bn/moving_mean"]) / np.sqrt(P[f"{scope}/bn/moving_variance"] + 1e-3) * P[f"{scope}/bn/gamma"] + P[f"{scope}/bn/beta"]
        net = np.maximum(z, 0.0)
    return net @ P["fc3/weights"] + P["fc3/biases"], pooled


def test_oracle_matches_a_plain_loop_transcription():
    from scanobjectnn_b200.synthetic import make_clouds
    b, n, k = 2, 32, 20
    xyz = make_clouds("ball", b, n, seed=3)
    d2 = ((xyz[:, :, None, :] - xyz[:, None, :, :]) ** 2).sum(-1)
    idx = np.argsort(d2, axis=-1, kind="stable")[:, :, :k].astype(np.int32)
    p = M.init_params(seed=5, device="cpu", randomize_bn=True)
    for key in list(p):                         # non-zero constant Taylor terms and conv biases, so that every term is pinned
        if key.endswith("/taylor/biases") or key.endswith("/conv/biases"):
            p[key] = torch.rand(p[key].shape, generator=torch.Generator().manual_seed(len(key))) - 0.5
    want_logits, want_pooled = _loop_forward(xyz, idx, p)
    logits, pooled, _ = so.forward(torch.from_numpy(xyz), torch.from_numpy(idx), p)
    np.testing.assert_allclose(pooled.numpy(), want_pooled, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(logits.numpy(), want_logits, rtol=1e-10, atol=1e-12)


def test_invalid_arguments_are_rejected_without_a_gpu():
    from scanobjectnn_b200 import _lib
    lib = _lib.load()
    null = C.c_void_p(0)
    ptrs = [null] * 9
    assert lib.psa_spider_conv_infer(-1, 16, 32, 20, 5, 64, *ptrs, null, 0, null) == -1
    assert lib.psa_spider_conv_infer(1, 16, 32, 0, 5, 64, *ptrs, null, 0, null) == -1            # k = 0
    assert lib.psa_spider_conv_infer(1, 16, 32, 33, 5, 64, *ptrs, null, 0, null) == -1           # k beyond the staged slots
    assert lib.psa_spider_conv_infer(1, 16, 32, 20, 0, 64, *ptrs, null, 0, null) == -1           # T = 0
    assert lib.psa_spider_conv_infer(1, 16, 32, 20, 5, 64, *ptrs, null, 0, null) == -1           # null buffers
    assert b"null buffer" in lib.psa_last_error()
    assert lib.psa_spider_conv_infer(0, 16, 32, 20, 5, 64, *ptrs, null, 0, null) == 0            # b = 0: no-op
    assert lib.psa_spider_conv_workspace_bytes(1, 16, 32, 33, 5, 64) == 0
    assert lib.psa_group_norm_affine(1, 16, 48, 32, C.c_float(1e-6), *[null] * 6, 1, null) == -1  # 32 groups do not divide 48
    assert lib.psa_group_norm_affine(1, 0, 32, 16, C.c_float(1e-6), *[null] * 6, 1, null) == -1
    assert lib.psa_topk_pool(1, 16, 32, 3, null, null, null, 1, null, 32, 0, null) == -2           # only k = 2
    assert lib.psa_topk_pool(1, 1, 32, 2, null, null, null, 1, null, 32, 0, null) == -1            # fewer points than k
    assert lib.psa_topk_pool(1, 16, 32, 2, null, null, null, 1, null, 48, 20, null) == -1          # channels past out_channels
