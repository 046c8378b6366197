"""Helpers for the -m gpu parity tests: torch<->numpy moves and ctypes calls into the compiled REFERENCE CUDA
kernels (oracle/_ref/libref_tfops.so) with torch device pointers."""
import ctypes as C

import numpy as np
import torch

from oracle import oracle as orc
from scanobjectnn_b200._lib import ptr


def cu(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.cuda()


def npy(t):
    return t.detach().cpu().numpy()


def ref_fps(xyz_t, m):
    b, n, _ = xyz_t.shape
    temp = torch.empty((32, n), dtype=torch.float32, device="cuda")
    out = torch.zeros((b, m), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    rc = orc.refgpu().ref_fps(b, n, m, ptr(xyz_t), ptr(temp), ptr(out), 1)
    assert rc == 0, rc
    return out


def ref_query_ball_point(radius, nsample, xyz1_t, xyz2_t, fill=0):
    b, n, _ = xyz1_t.shape
    m = xyz2_t.shape[1]
    idx = torch.full((b, m, nsample), fill, dtype=torch.int32, device="cuda")
    cnt = torch.zeros((b, m), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    rc = orc.refgpu().ref_query_ball_point(b, n, m, C.c_float(radius), nsample, ptr(xyz1_t), ptr(xyz2_t), ptr(idx), ptr(cnt), 1)
    assert rc == 0, rc
    return idx, cnt


def ref_group_point(points_t, idx_t):
    b, n, c = points_t.shape
    _, m, k = idx_t.shape
    out = torch.empty((b, m, k, c), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    rc = orc.refgpu().ref_group_point(b, n, c, m, k, ptr(points_t), ptr(idx_t), ptr(out), 1)
    assert rc == 0, rc
    return out


def ref_selection_sort(k, dist_t):
    b, m, n = dist_t.shape
    outi = torch.empty((b, m, n), dtype=torch.int32, device="cuda")
    out = torch.empty((b, m, n), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    rc = orc.refgpu().ref_selection_sort(b, n, m, k, ptr(dist_t), ptr(outi), ptr(out), 1)
    assert rc == 0, rc
    return outi, out


def ref_gather_point(inp_t, idx_t):
    b, n, _ = inp_t.shape
    m = idx_t.shape[1]
    out = torch.empty((b, m, 3), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    rc = orc.refgpu().ref_gather_point(b, n, m, ptr(inp_t), ptr(idx_t), ptr(out), 1)
    assert rc == 0, rc
    return out


CONTRACT_TOL = 1e-5   # BASELINE.json north_star: grouped-MLP activations within 1e-5 (fp32)


def contract_close(got, want, what=""):
    """The floating-point contract of the path.  Activations of magnitude <= 1: max|got - want| < 1e-5 ABSOLUTE.  Larger
    activations: 1e-5 relative to the largest activation (fp32 itself resolves no better), with the scale printed so the
    log shows which bound was applied.  Returns the error."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    err = float(np.abs(got - want).max()) if want.size else 0.0
    scale = float(np.abs(want).max()) if want.size else 0.0
    if scale <= 1.0:
        assert err < CONTRACT_TOL, f"{what}: max|err| = {err:.3e} >= 1e-5 absolute (max|act| = {scale:.3f})"
    else:
        print(f"[contract] {what}: max|act| = {scale:.3f} > 1 -> bound 1e-5 * {scale:.3f}; max|err| = {err:.3e}")
        assert err < CONTRACT_TOL * scale, f"{what}: max|err| = {err:.3e} >= 1e-5 * max|act| ({scale:.3f})"
    return err
