"""ctypes/numpy face of the CPU checker (oracle/liboracle.so) and of the compiled reference
(oracle/_ref/libref_cpu.so = the reference's own CPU code, oracle/_ref/libref_tfops.so = the reference's
own CUDA kernels for sm_90a).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
``--impl reference`` leg.  Nothing under scanobjectnn_b200/ may import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_F = np.float32
_I = np.int32


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f32(a):
    return np.ascontiguousarray(a, dtype=_F)


def _i32(a):
    return np.ascontiguousarray(a, dtype=_I)


def build(ref: bool | None = None) -> None:
    """(Re)build liboracle.so; also oracle/_ref when the reference checkout is present."""
    subprocess.run(["make", "-C", _HERE, "-s"], check=True)
    if ref is None:
        ref = os.path.isdir("/root/reference/pointnet2/tf_ops")
    if ref:
        subprocess.run(["make", "-C", _HERE, "-s", "ref"], check=True)


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        path = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(path):
            build(ref=False)
        _lib = C.CDLL(path)
    return _lib


# ---------------------------------------------------------------------------------------------
# this repo's restatement
# ---------------------------------------------------------------------------------------------
def fps(xyz, m):
    xyz = _f32(xyz); b, n, _ = xyz.shape
    out = np.zeros((b, m), _I)
    lib().orc_fps(b, n, m, _p(xyz), _p(out))
    return out


def gather_point(inp, idx):
    inp = _f32(inp); idx = _i32(idx); b, n, _ = inp.shape; m = idx.shape[1]
    out = np.empty((b, m, 3), _F)
    lib().orc_gather_point(b, n, m, _p(inp), _p(idx), _p(out))
    return out


def gather_point_grad(inp_shape, idx, out_g):
    idx = _i32(idx); out_g = _f32(out_g); b, n, _ = inp_shape; m = idx.shape[1]
    g = np.empty((b, n, 3), _F)
    lib().orc_gather_point_grad(b, n, m, _p(out_g), _p(idx), _p(g))
    return g


def query_ball_point(radius, nsample, xyz1, xyz2, contract=True, fill=0):
    xyz1 = _f32(xyz1); xyz2 = _f32(xyz2); b, n, _ = xyz1.shape; m = xyz2.shape[1]
    idx = np.full((b, m, nsample), fill, _I)
    cnt = np.zeros((b, m), _I)
    lib().orc_query_ball_point(b, n, m, C.c_float(radius), nsample, _p(xyz1), _p(xyz2), _p(idx), _p(cnt),
                               1 if contract else 0)
    return idx, cnt


def group_point(points, idx):
    points = _f32(points); idx = _i32(idx); b, n, c = points.shape; _, m, k = idx.shape
    out = np.empty((b, m, k, c), _F)
    lib().orc_group_point(b, n, c, m, k, _p(points), _p(idx), _p(out))
    return out


def group_point_grad(points_shape, idx, grad_out):
    idx = _i32(idx); grad_out = _f32(grad_out); b, n, c = points_shape; _, m, k = idx.shape
    g = np.empty((b, n, c), _F)
    lib().orc_group_point_grad(b, n, c, m, k, _p(grad_out), _p(idx), _p(g))
    return g


def selection_sort(k, dist):
    dist = _f32(dist); b, m, n = dist.shape
    outi = np.empty((b, m, n), _I); out = np.empty((b, m, n), _F)
    lib().orc_selection_sort(b, n, m, k, _p(dist), _p(outi), _p(out))
    return outi, out


def knn_point(k, xyz1, xyz2):
    """tf_grouping.py:49-74 -> (val (b,m,k), idx (b,m,k))"""
    xyz1 = _f32(xyz1); xyz2 = _f32(xyz2); b, n, c = xyz1.shape; m = xyz2.shape[1]
    dist = np.empty((b, m, n), _F)
    lib().orc_knn_point_dist(b, n, m, c, _p(xyz1), _p(xyz2), _p(dist))
    outi, out = selection_sort(k, dist)
    return out[:, :, :k].copy(), outi[:, :, :k].copy()


def three_nn(xyz1, xyz2):
    xyz1 = _f32(xyz1); xyz2 = _f32(xyz2); b, n, _ = xyz1.shape; m = xyz2.shape[1]
    dist = np.empty((b, n, 3), _F); idx = np.empty((b, n, 3), _I)
    lib().orc_three_nn(b, n, m, _p(xyz1), _p(xyz2), _p(dist), _p(idx))
    return dist, idx


def three_interpolate(points, idx, weight):
    points = _f32(points); idx = _i32(idx); weight = _f32(weight)
    b, m, c = points.shape; n = idx.shape[1]
    out = np.empty((b, n, c), _F)
    lib().orc_three_interpolate(b, m, c, n, _p(points), _p(idx), _p(weight), _p(out))
    return out


def three_interpolate_grad(points_shape, idx, weight, grad_out):
    idx = _i32(idx); weight = _f32(weight); grad_out = _f32(grad_out)
    b, m, c = points_shape; n = idx.shape[1]
    g = np.empty((b, m, c), _F)
    lib().orc_three_interpolate_grad(b, n, c, m, _p(grad_out), _p(idx), _p(weight), _p(g))
    return g


def three_weights(dist):
    dist = _f32(dist)
    w = np.empty_like(dist)
    lib().orc_three_weights(int(dist.size // 3), _p(dist), _p(w))
    return w


def dgcnn_knn(x, k, want_adj=False):
    x = _f32(x); b, n, c = x.shape
    idx = np.empty((b, n, k), _I)
    adj = np.empty((b, n, n), _F) if want_adj else None
    lib().orc_dgcnn_knn(b, n, c, k, _p(x), _p(adj) if want_adj else None, _p(idx))
    return (idx, adj) if want_adj else idx


def topk_smallest(adj, k):
    adj = _f32(adj); b, n, n2 = adj.shape
    idx = np.empty((b, n, k), _I)
    lib().orc_topk_smallest(b * n, n2, k, _p(adj), _p(idx))
    return idx


# ---------------------------------------------------------------------------------------------
# the reference's own CPU code (oracle/_ref/libref_cpu.so) -- present after `make -C oracle ref`
# ---------------------------------------------------------------------------------------------
_refcpu = None


def refcpu_available() -> bool:
    return os.path.exists(os.path.join(_HERE, "_ref", "libref_cpu.so"))


def refcpu() -> C.CDLL:
    global _refcpu
    if _refcpu is None:
        _refcpu = C.CDLL(os.path.join(_HERE, "_ref", "libref_cpu.so"))
    return _refcpu


def refcpu_query_ball_point(radius, nsample, xyz1, xyz2, fill=0):
    xyz1 = _f32(xyz1); xyz2 = _f32(xyz2); b, n, _ = xyz1.shape; m = xyz2.shape[1]
    idx = np.full((b, m, nsample), fill, _I)
    refcpu().refcpu_query_ball_point(b, n, m, C.c_float(radius), nsample, _p(xyz1), _p(xyz2), _p(idx))
    return idx


def refcpu_group_point(points, idx):
    points = _f32(points); idx = _i32(idx); b, n, c = points.shape; _, m, k = idx.shape
    out = np.empty((b, m, k, c), _F)
    refcpu().refcpu_group_point(b, n, c, m, k, _p(points), _p(idx), _p(out))
    return out


def refcpu_group_point_grad(points_shape, idx, grad_out):
    idx = _i32(idx); grad_out = _f32(grad_out); b, n, c = points_shape; _, m, k = idx.shape
    g = np.zeros((b, n, c), _F)
    refcpu().refcpu_group_point_grad(b, n, c, m, k, _p(grad_out), _p(idx), _p(g))
    return g


def refcpu_selection_sort(k, dist):
    dist = _f32(dist); b, m, n = dist.shape
    outi = np.zeros((b, m, n), _I); out = np.zeros((b, m, n), _F)
    refcpu().refcpu_selection_sort(b, n, m, k, _p(dist), _p(outi), _p(out))
    return outi, out


def refcpu_three_nn(xyz1, xyz2):
    xyz1 = _f32(xyz1); xyz2 = _f32(xyz2); b, n, _ = xyz1.shape; m = xyz2.shape[1]
    dist = np.empty((b, n, 3), _F); idx = np.empty((b, n, 3), _I)
    refcpu().refcpu_three_nn(b, n, m, _p(xyz1), _p(xyz2), _p(dist), _p(idx))
    return dist, idx


def refcpu_three_interpolate(points, idx, weight):
    points = _f32(points); idx = _i32(idx); weight = _f32(weight)
    b, m, c = points.shape; n = idx.shape[1]
    out = np.empty((b, n, c), _F)
    refcpu().refcpu_three_interpolate(b, m, c, n, _p(points), _p(idx), _p(weight), _p(out))
    return out


def refcpu_three_interpolate_grad(points_shape, idx, weight, grad_out):
    idx = _i32(idx); weight = _f32(weight); grad_out = _f32(grad_out)
    b, m, c = points_shape; n = idx.shape[1]
    g = np.zeros((b, m, c), _F)
    refcpu().refcpu_three_interpolate_grad(b, n, c, m, _p(grad_out), _p(idx), _p(weight), _p(g))
    return g


# ---------------------------------------------------------------------------------------------
# the reference's own CUDA kernels (oracle/_ref/libref_tfops.so) -- device pointers, needs a GPU
# ---------------------------------------------------------------------------------------------
_refgpu = None


def refgpu_available() -> bool:
    return os.path.exists(os.path.join(_HERE, "_ref", "libref_tfops.so"))


def refgpu() -> C.CDLL:
    global _refgpu
    if _refgpu is None:
        _refgpu = C.CDLL(os.path.join(_HERE, "_ref", "libref_tfops.so"))
    return _refgpu
