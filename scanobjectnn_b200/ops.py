"""PyTorch-tensor face of libpsa.so: the reference's op names and argument order on CUDA tensors.

Mirrors pointnet2/tf_ops/{sampling/tf_sampling.py, grouping/tf_grouping.py, 3d_interpolation/tf_interpolate.py}
and dgcnn/utils/tf_util.py:638-706.  Every function validates like the reference's OP_REQUIRES (-> ValueError),
then calls the C ABI (include/psa.h) on the current torch CUDA stream with raw device pointers.  Torch is
plumbing here (allocation, streams, autograd glue); all arithmetic happens in the hand-written kernels.
There is no CPU path: CPU tensors raise.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import PsaMlp, check
from ._lib import ptr as _ptr
from ._lib import stream as _stream

__all__ = [
    "farthest_point_sample", "gather_point", "query_ball_point", "group_point", "select_top_k", "knn_point",
    "three_nn", "three_interpolate", "three_nn_interpolate", "pairwise_distance", "knn", "knn_graph",
    "get_edge_feature", "farthest_point_sample_and_gather", "MlpParams", "shared_mlp", "shared_mlp_grouped", "sa_module_infer",
    "edgeconv_infer", "sa_conv1_prebn", "pool_rows", "sa_group_all_infer", "set_mlp_mode", "get_mlp_mode",
    "spider_conv", "group_norm_affine", "topk_pool", "fisher_vector", "conv3d", "pool3d", "knn_dilated", "xconv_core",
    "dense_elu_affine", "conv3d_bwd_weight", "conv3d_bwd_data", "conv3d_bwd_macs", "pool3d_max_train", "pool3d_bwd",
    "elu_bn_dy", "bn_affine_rows", "xconv_depthwise_bwd",
]


def _dev(t: torch.Tensor, dtype: torch.dtype, name: str, ndim: int | None = None) -> torch.Tensor:
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name}: expected a torch.Tensor")
    if not t.is_cuda:
        raise RuntimeError(f"{name}: expected a CUDA tensor (scanobjectnn_b200 has no CPU path)")
    if t.dtype != dtype:
        raise TypeError(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if ndim is not None and t.dim() != ndim:
        raise ValueError(f"{name}: expected a {ndim}-D tensor, got shape {tuple(t.shape)}")
    return t.contiguous()


def _scatter_ws(b: int, n_dst: int, entries: int, device) -> tuple[torch.Tensor, C.c_size_t]:
    """Scratch for the ordered scatter-add gradients (psa_scatter_workspace_bytes)."""
    need = int(_lib.load().psa_scatter_workspace_bytes(b, n_dst, entries))
    return torch.empty((need,), dtype=torch.uint8, device=device), C.c_size_t(need)


# ------------------------------------------------------------------------------------------------
# sampling
# ------------------------------------------------------------------------------------------------
def farthest_point_sample_and_gather(npoint: int, inp: torch.Tensor):
    """FPS with the gather_point of the result fused: -> (idx (B,npoint) int32, new_xyz (B,npoint,3))."""
    inp = _dev(inp, torch.float32, "inp", 3)
    if inp.shape[2] != 3:
        raise ValueError("FarthestPointSample expects (batch_size,num_points,3) inp shape")  # tf_sampling.cpp:105
    b, n, _ = inp.shape
    idx = torch.empty((b, npoint), dtype=torch.int32, device=inp.device)
    new_xyz = torch.empty((b, npoint, 3), dtype=torch.float32, device=inp.device)
    check(_lib.load().psa_farthest_point_sample(b, n, npoint, _ptr(inp), _ptr(idx), _ptr(new_xyz), _stream()),
          "farthest_point_sample")
    return idx, new_xyz


def farthest_point_sample(npoint: int, inp: torch.Tensor) -> torch.Tensor:
    """tf_sampling.farthest_point_sample (tf_sampling.py:49-58): inp (B,N,3) f32 -> (B,npoint) int32."""
    inp = _dev(inp, torch.float32, "inp", 3)
    if inp.shape[2] != 3:
        raise ValueError("FarthestPointSample expects (batch_size,num_points,3) inp shape")
    b, n, _ = inp.shape
    idx = torch.empty((b, npoint), dtype=torch.int32, device=inp.device)
    check(_lib.load().psa_farthest_point_sample(b, n, npoint, _ptr(inp), _ptr(idx), _ptr(None), _stream()),
          "farthest_point_sample")
    return idx


class _GatherPoint(torch.autograd.Function):
    @staticmethod
    def forward(ctx, inp, idx):
        b, n, _ = inp.shape
        m = idx.shape[1]
        out = torch.empty((b, m, 3), dtype=torch.float32, device=inp.device)
        check(_lib.load().psa_gather_point(b, n, m, _ptr(inp), _ptr(idx), _ptr(out), _stream()), "gather_point")
        ctx.save_for_backward(idx)
        ctx.n = n
        return out

    @staticmethod
    def backward(ctx, out_g):
        (idx,) = ctx.saved_tensors
        out_g = out_g.contiguous()
        b, m, _ = out_g.shape
        inp_g = torch.empty((b, ctx.n, 3), dtype=torch.float32, device=out_g.device)
        ws, nbytes = _scatter_ws(b, ctx.n, m, out_g.device)
        check(_lib.load().psa_gather_point_grad(b, ctx.n, m, _ptr(out_g), _ptr(idx), _ptr(inp_g), _ptr(ws), nbytes, _stream()),
              "gather_point_grad")
        return inp_g, None


def gather_point(inp: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """tf_sampling.gather_point (tf_sampling.py:30-38): inp (B,N,3), idx (B,M) int32 -> (B,M,3); differentiable
    w.r.t. inp (GatherPointGrad, tf_sampling.py:44-48)."""
    inp = _dev(inp, torch.float32, "inp", 3)
    idx = _dev(idx, torch.int32, "idx", 2)
    if inp.shape[2] != 3:
        raise ValueError("GatherPoint expects (batch_size,num_points,3) inp shape")          # tf_sampling.cpp:134
    if idx.shape[0] != inp.shape[0]:
        raise ValueError("GatherPoint expects (batch_size,num_result) idx shape")            # tf_sampling.cpp:138
    return _GatherPoint.apply(inp, idx)


# ------------------------------------------------------------------------------------------------
# grouping
# ------------------------------------------------------------------------------------------------
def query_ball_point(radius: float, nsample: int, xyz1: torch.Tensor, xyz2: torch.Tensor):
    """tf_grouping.query_ball_point (tf_grouping.py:9-21): xyz1 (B,N,3) dataset, xyz2 (B,M,3) queries ->
    (idx (B,M,nsample) int32, pts_cnt (B,M) int32)."""
    if not radius > 0:
        raise ValueError("QueryBallPoint expects positive radius")                           # tf_grouping.cpp:71
    if not nsample > 0:
        raise ValueError("QueryBallPoint expects positive nsample")                          # tf_grouping.cpp:74
    xyz1 = _dev(xyz1, torch.float32, "xyz1", 3)
    xyz2 = _dev(xyz2, torch.float32, "xyz2", 3)
    if xyz1.shape[2] != 3:
        raise ValueError("QueryBallPoint expects (batch_size, ndataset, 3) xyz1 shape.")     # tf_grouping.cpp:79
    if xyz2.shape[2] != 3 or xyz2.shape[0] != xyz1.shape[0]:
        raise ValueError("QueryBallPoint expects (batch_size, npoint, 3) xyz2 shape.")       # tf_grouping.cpp:84
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    idx = torch.empty((b, m, nsample), dtype=torch.int32, device=xyz1.device)
    cnt = torch.empty((b, m), dtype=torch.int32, device=xyz1.device)
    check(_lib.load().psa_query_ball_point(b, n, m, C.c_float(radius), nsample, _ptr(xyz1), _ptr(xyz2), _ptr(idx),
                                           _ptr(cnt), _stream()), "query_ball_point")
    return idx, cnt


class _GroupPoint(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, idx):
        b, n, c = points.shape
        _, m, k = idx.shape
        out = torch.empty((b, m, k, c), dtype=torch.float32, device=points.device)
        check(_lib.load().psa_group_point(b, n, c, m, k, _ptr(points), _ptr(idx), _ptr(out), _stream()), "group_point")
        ctx.save_for_backward(idx)
        ctx.shape = (b, n, c)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        (idx,) = ctx.saved_tensors
        b, n, c = ctx.shape
        _, m, k = idx.shape
        grad_out = grad_out.contiguous()
        g = torch.empty((b, n, c), dtype=torch.float32, device=grad_out.device)
        ws, nbytes = _scatter_ws(b, n, m * k, grad_out.device)
        check(_lib.load().psa_group_point_grad(b, n, c, m, k, _ptr(grad_out), _ptr(idx), _ptr(g), _ptr(ws), nbytes, _stream()),
              "group_point_grad")
        return g, None


def group_point(points: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """tf_grouping.group_point (tf_grouping.py:34-42): points (B,N,C), idx (B,M,K) -> (B,M,K,C); differentiable
    w.r.t. points (GroupPointGrad, tf_grouping.py:43-47)."""
    points = _dev(points, torch.float32, "points", 3)
    idx = _dev(idx, torch.int32, "idx", 3)
    if idx.shape[0] != points.shape[0]:
        raise ValueError("GroupPoint expects (batch_size, npoints, nsample) idx shape")      # tf_grouping.cpp:157
    return _GroupPoint.apply(points, idx)


def select_top_k(k: int, dist: torch.Tensor):
    """tf_grouping.select_top_k (tf_grouping.py:23-33): dist (B,M,N) -> (idx (B,M,N) int32, dist_out (B,M,N));
    the first k slots of each row are the k smallest (SelectionSort semantics, ties by current position)."""
    if not k > 0:
        raise ValueError("SelectionSort expects positive k")                                 # tf_grouping.cpp:113
    dist = _dev(dist, torch.float32, "dist", 3)
    b, m, n = dist.shape
    outi = torch.empty((b, m, n), dtype=torch.int32, device=dist.device)
    out = torch.empty((b, m, n), dtype=torch.float32, device=dist.device)
    check(_lib.load().psa_selection_sort(b, n, m, k, _ptr(dist), _ptr(outi), _ptr(out), _stream()), "select_top_k")
    return outi, out


def knn_point(k: int, xyz1: torch.Tensor, xyz2: torch.Tensor):
    """tf_grouping.knn_point (tf_grouping.py:49-74): xyz1 (B,N,C) dataset, xyz2 (B,M,C) queries ->
    (val (B,M,k), idx (B,M,k) int32) without building the (B,M,N) matrices."""
    xyz1 = _dev(xyz1, torch.float32, "xyz1", 3)
    xyz2 = _dev(xyz2, torch.float32, "xyz2", 3)
    if xyz1.shape[0] != xyz2.shape[0] or xyz1.shape[2] != xyz2.shape[2]:
        raise ValueError("knn_point expects xyz1 (b,n,c) and xyz2 (b,m,c)")
    b, n, c = xyz1.shape
    m = xyz2.shape[1]
    val = torch.empty((b, m, k), dtype=torch.float32, device=xyz1.device)
    idx = torch.empty((b, m, k), dtype=torch.int32, device=xyz1.device)
    check(_lib.load().psa_knn_point(b, n, m, c, k, _ptr(xyz1), _ptr(xyz2), _ptr(val), _ptr(idx), _stream()), "knn_point")
    return val, idx


# ------------------------------------------------------------------------------------------------
# input pipeline (data_utils.py / provider.py of the reference, numpy on the host there)
# ------------------------------------------------------------------------------------------------
def augment_batch(src: torch.Tensor, n: int | None = None, *, perm=None, angles=None, scale=None, shift=None, noise=None,
                  sigma: float = 0.01, clip: float = 0.05, drop=None, center: bool = False, normalize: bool = False) -> torch.Tensor:
    """center_data / normalize_data (data_utils.py:133-168) over the whole source cloud, the epoch's point subset
    (get_current_data_h5, data_utils.py:171-186: ``perm[:n]``, the same for every cloud), then per batch
    rotate_point_cloud about the up axis (provider.py:34-52, ``angles`` (B,) radians) and jitter_point_cloud
    (provider.py:189-200, ``noise`` (B,n,3) standard normal) -- the composition the training scripts run
    (pointnet2/train.py:246-252), same order and precisions, in one launch.
    Optional extras, each with its provider.py arithmetic but in THIS kernel's fixed order (the reference only composes them
    in a commented-out block, dgcnn/train.py:274-278, which jitters BEFORE scaling): dropped slots (``drop`` (B,n) bool,
    provider.py:229-236) read source point 0, then rotate -> scale -> shift (provider.py:202-227) -> jitter; every output
    slot gets its own jitter noise, so dropped slots equal point 0 only up to that noise.
    src (B,N_src,3) float32 -> (B,n,3).  The random numbers are arguments: draw them with ``draw_augmentation``."""
    src = _dev(src, torch.float32, "src", 3)
    if src.shape[2] != 3:
        raise ValueError("augment_batch expects (batch, num_points, 3) input")
    b, n_src, _ = src.shape
    n = n_src if n is None else int(n)
    dev = src.device
    cs = None
    if angles is not None:
        if isinstance(angles, torch.Tensor) and angles.is_cuda:                        # stay on the device: no host sync per batch
            ang = angles.to(torch.float64).reshape(b)
        else:
            ang = torch.as_tensor(angles, dtype=torch.float64).reshape(b)              # host libm, bit-identical to numpy's
        cs = torch.stack([torch.cos(ang), torch.sin(ang)], dim=1).contiguous().to(dev)  # cos / sin in float64 like numpy
    perm_t = None if perm is None else _dev(torch.as_tensor(perm, device=dev), torch.int32, "perm", 1)
    if perm_t is not None and perm_t.numel() < n:
        raise ValueError("augment_batch: perm is shorter than n")
    if perm_t is None and n > n_src:
        raise ValueError("augment_batch: n exceeds the source cloud")
    scale_t = None if scale is None else _dev(torch.as_tensor(scale, device=dev), torch.float32, "scale", 1)
    shift_t = None if shift is None else _dev(torch.as_tensor(shift, device=dev), torch.float32, "shift", 2)
    noise_t = None if noise is None else _dev(torch.as_tensor(noise, device=dev), torch.float32, "noise", 3)
    drop_t = None if drop is None else torch.as_tensor(drop, device=dev).to(torch.uint8).contiguous()
    if noise_t is not None and not clip > 0:
        raise ValueError("jitter_point_cloud: clip must be positive")                  # provider.py:196 assert(clip > 0)
    out = torch.empty((b, n, 3), dtype=torch.float32, device=dev)
    check(_lib.load().psa_augment_batch(b, n_src, n, _ptr(src), _ptr(perm_t), _ptr(cs), _ptr(scale_t), _ptr(shift_t), _ptr(noise_t),
                                        C.c_double(sigma), C.c_double(clip), _ptr(drop_t), int(bool(center)), int(bool(normalize)),
                                        _ptr(out), _stream()), "augment_batch")
    return out


def draw_augmentation(b: int, n_src: int, n: int, device, generator: torch.Generator | None = None, jitter: bool = True):
    """The random numbers of one training batch as the reference draws them (one point subset per epoch, one angle per
    cloud, one normal sample per coordinate), on the device: dict for ``augment_batch(**...)``."""
    g = generator
    perm = torch.randperm(n_src, device=device, generator=g)[:n].to(torch.int32)
    angles = torch.rand(b, device=device, generator=g, dtype=torch.float64) * (2.0 * 3.141592653589793)
    out = {"perm": perm, "angles": angles}
    if jitter:
        out["noise"] = torch.randn((b, n, 3), device=device, generator=g)
    return out


# ------------------------------------------------------------------------------------------------
# 3d interpolation
# ------------------------------------------------------------------------------------------------
def three_nn(xyz1: torch.Tensor, xyz2: torch.Tensor):
    """tf_interpolate.three_nn (tf_interpolate.py:9-18): xyz1 (B,N,3) unknown, xyz2 (B,M,3) known ->
    (dist (B,N,3) squared, idx (B,N,3) int32)."""
    xyz1 = _dev(xyz1, torch.float32, "xyz1", 3)
    xyz2 = _dev(xyz2, torch.float32, "xyz2", 3)
    if xyz1.shape[2] != 3:
        raise ValueError("ThreeNN expects (b,n,3) xyz1 shape")                               # tf_interpolate.cpp:164
    if xyz2.shape[2] != 3 or xyz2.shape[0] != xyz1.shape[0]:
        raise ValueError("ThreeNN expects (b,m,3) xyz2 shape")                               # tf_interpolate.cpp:169
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    dist = torch.empty((b, n, 3), dtype=torch.float32, device=xyz1.device)
    idx = torch.empty((b, n, 3), dtype=torch.int32, device=xyz1.device)
    check(_lib.load().psa_three_nn(b, n, m, _ptr(xyz1), _ptr(xyz2), _ptr(dist), _ptr(idx), _stream()), "three_nn")
    return dist, idx


class _ThreeInterpolate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, idx, weight):
        b, m, c = points.shape
        n = idx.shape[1]
        out = torch.empty((b, n, c), dtype=torch.float32, device=points.device)
        check(_lib.load().psa_three_interpolate(b, m, c, n, _ptr(points), _ptr(idx), _ptr(weight), _ptr(out), _stream()),
              "three_interpolate")
        ctx.save_for_backward(idx, weight)
        ctx.shape = (b, m, c)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        idx, weight = ctx.saved_tensors
        b, m, c = ctx.shape
        n = idx.shape[1]
        grad_out = grad_out.contiguous()
        g = torch.empty((b, m, c), dtype=torch.float32, device=grad_out.device)
        ws, nbytes = _scatter_ws(b, m, 3 * n, grad_out.device)
        check(_lib.load().psa_three_interpolate_grad(b, n, c, m, _ptr(grad_out), _ptr(idx), _ptr(weight), _ptr(g), _ptr(ws), nbytes,
                                                     _stream()), "three_interpolate_grad")
        return g, None, None


def three_interpolate(points: torch.Tensor, idx: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """tf_interpolate.three_interpolate (tf_interpolate.py:20-35): points (B,M,C), idx (B,N,3), weight (B,N,3) ->
    (B,N,C); differentiable w.r.t. points (ThreeInterpolateGrad)."""
    points = _dev(points, torch.float32, "points", 3)
    idx = _dev(idx, torch.int32, "idx", 3)
    weight = _dev(weight, torch.float32, "weight", 3)
    if idx.shape[0] != points.shape[0] or idx.shape[2] != 3:
        raise ValueError("ThreeInterpolate expects (b,n,3) idx shape")                       # tf_interpolate.cpp:199
    if weight.shape != idx.shape:
        raise ValueError("ThreeInterpolate expects (b,n,3) weight shape")                    # tf_interpolate.cpp:202
    return _ThreeInterpolate.apply(points, idx, weight)


def three_nn_interpolate(xyz1, xyz2, points2, return_aux: bool = False):
    """pointnet_fp_module's interpolation (pointnet_util.py:211-216) in one launch -> (B,N,C)
    [, dist, idx, weight when return_aux]."""
    xyz1 = _dev(xyz1, torch.float32, "xyz1", 3)
    xyz2 = _dev(xyz2, torch.float32, "xyz2", 3)
    points2 = _dev(points2, torch.float32, "points2", 3)
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    c = points2.shape[2]
    if points2.shape[0] != b or points2.shape[1] != m or xyz2.shape[0] != b:
        raise ValueError("three_nn_interpolate expects xyz2 (b,m,3) and points2 (b,m,c)")
    out = torch.empty((b, n, c), dtype=torch.float32, device=xyz1.device)
    dist = idx = weight = None
    if return_aux:
        dist = torch.empty((b, n, 3), dtype=torch.float32, device=xyz1.device)
        idx = torch.empty((b, n, 3), dtype=torch.int32, device=xyz1.device)
        weight = torch.empty((b, n, 3), dtype=torch.float32, device=xyz1.device)
    check(_lib.load().psa_three_nn_interpolate(b, n, m, c, _ptr(xyz1), _ptr(xyz2), _ptr(points2), _ptr(out), _ptr(dist),
                                               _ptr(idx), _ptr(weight), _stream()), "three_nn_interpolate")
    return (out, dist, idx, weight) if return_aux else out


# ------------------------------------------------------------------------------------------------
# dgcnn graph functions
# ------------------------------------------------------------------------------------------------
def _squeeze_pc(point_cloud: torch.Tensor) -> torch.Tensor:
    # dgcnn/utils/tf_util.py:647-650: tf.squeeze, re-expanding a batch of one
    og = point_cloud.shape[0]
    pc = point_cloud.squeeze()
    if og == 1:
        pc = pc.unsqueeze(0)
    if pc.dim() != 3:
        raise ValueError(f"expected (B,N,C) or (B,N,1,C), got {tuple(point_cloud.shape)}")
    return pc


def pairwise_distance(point_cloud: torch.Tensor) -> torch.Tensor:
    """dgcnn tf_util.pairwise_distance (tf_util.py:638-657): (B,N,C) or (B,N,1,C) -> (B,N,N)."""
    pc = _dev(_squeeze_pc(point_cloud), torch.float32, "point_cloud", 3)
    b, n, c = pc.shape
    adj = torch.empty((b, n, n), dtype=torch.float32, device=pc.device)
    check(_lib.load().psa_pairwise_distance(b, n, c, _ptr(pc), _ptr(adj), _stream()), "pairwise_distance")
    return adj


def knn(adj_matrix: torch.Tensor, k: int = 20) -> torch.Tensor:
    """dgcnn tf_util.knn (tf_util.py:660-671): (B,N,N) -> nn_idx (B,N,k) int32, ascending distance, self included."""
    adj = _dev(adj_matrix, torch.float32, "adj_matrix", 3)
    b, n, ncols = adj.shape
    nn_idx = torch.empty((b, n, k), dtype=torch.int32, device=adj.device)
    check(_lib.load().psa_knn_topk(b, n, ncols, k, _ptr(adj), _ptr(nn_idx), _stream()), "knn")
    return nn_idx


def knn_graph(point_cloud: torch.Tensor, k: int = 20) -> torch.Tensor:
    """knn(pairwise_distance(point_cloud), k) fused -- no (B,N,N) matrix."""
    pc = _dev(_squeeze_pc(point_cloud), torch.float32, "point_cloud", 3)
    b, n, c = pc.shape
    nn_idx = torch.empty((b, n, k), dtype=torch.int32, device=pc.device)
    lib = _lib.load()
    # tensor-core contraction + exact refine (csrc/knn_tc.cu) where it applies, the fp32 kernel otherwise: same indices
    need = lib.psa_knn_graph_workspace_bytes(b, n, c, k)
    ws = torch.empty((need + 3) // 4, dtype=torch.float32, device=pc.device) if need else None
    check(lib.psa_knn_graph_ws(b, n, c, k, _ptr(pc), _ptr(nn_idx), _ptr(ws), C.c_size_t(need), _stream()), "knn_graph")
    return nn_idx


def get_edge_feature(point_cloud: torch.Tensor, nn_idx: torch.Tensor, k: int = 20) -> torch.Tensor:
    """dgcnn tf_util.get_edge_feature (tf_util.py:674-706): (B,N,C)/(B,N,1,C), nn_idx (B,N,k) -> (B,N,k,2C)."""
    pc = _dev(_squeeze_pc(point_cloud), torch.float32, "point_cloud", 3)
    nn_idx = _dev(nn_idx, torch.int32, "nn_idx", 3)
    b, n, c = pc.shape
    if nn_idx.shape[0] != b or nn_idx.shape[1] != n or nn_idx.shape[2] != k:
        raise ValueError("get_edge_feature expects nn_idx (B,N,k)")
    out = torch.empty((b, n, k, 2 * c), dtype=torch.float32, device=pc.device)
    check(_lib.load().psa_get_edge_feature(b, n, c, k, _ptr(pc), _ptr(nn_idx), _ptr(out), _stream()), "get_edge_feature")
    return out


# ------------------------------------------------------------------------------------------------
# grouped shared MLP
# ------------------------------------------------------------------------------------------------
class MlpParams:
    """Device-side description of a shared MLP for the fused kernels (struct psa_mlp in include/psa.h).

    layers: list of (weight (C_in,C_out), scale (C_out) or None, shift (C_out), relu: bool) -- conv bias and
    inference-mode batch norm already folded by the caller (see pointnet_util.fold_conv_bn)."""

    def __init__(self, layers):
        if not 1 <= len(layers) <= _lib.PSA_MAX_MLP_LAYERS:
            raise ValueError(f"a fused MLP has 1..{_lib.PSA_MAX_MLP_LAYERS} layers, got {len(layers)}")
        self._keep = []
        s = PsaMlp()
        s.n_layers = len(layers)
        for l, (w, scale, shift, relu) in enumerate(layers):
            w = _dev(w, torch.float32, f"weight[{l}]", 2)
            shift = _dev(shift, torch.float32, f"shift[{l}]", 1)
            if scale is not None:
                scale = _dev(scale, torch.float32, f"scale[{l}]", 1)
            cin, cout = w.shape
            if l == 0:
                s.channels[0] = cin
            elif s.channels[l] != cin:
                raise ValueError(f"layer {l}: C_in={cin} does not chain with previous C_out={s.channels[l]}")
            if shift.numel() != cout or (scale is not None and scale.numel() != cout):
                raise ValueError(f"layer {l}: scale/shift must have {cout} entries")
            s.channels[l + 1] = cout
            s.weight[l] = w.data_ptr()
            s.scale[l] = 0 if scale is None else scale.data_ptr()
            s.shift[l] = shift.data_ptr()
            s.relu[l] = 1 if relu else 0
            self._keep += [w, scale, shift]
        self.struct = s
        self.channels = [s.channels[i] for i in range(len(layers) + 1)]
        self._weights = [w for (w, _, _, _) in [(self._keep[3 * i], None, None, None) for i in range(len(layers))]]
        self._prepared = {}

    @property
    def ref(self):
        return C.byref(self.struct)

    def prepared(self, usage: int, rows: int, pool_k: int = 1, c: int = 0, nsample: int = 0):
        """byref of a copy of the struct whose tensor-core weight images were built ONCE (inference: the weights do not
        change between calls), so the entry points skip the per-call prep kernels.  Keyed by what the C side says it
        will use for this (usage, shape)."""
        lib = _lib.load()
        L = self.struct.n_layers
        nt = (C.c_int * _lib.PSA_MAX_MLP_LAYERS)()
        row0 = (C.c_int * _lib.PSA_MAX_MLP_LAYERS)()
        nbytes = (C.c_size_t * _lib.PSA_MAX_MLP_LAYERS)()
        check(lib.psa_mlp_image_plan(usage, rows, pool_k, c, nsample, self.ref, nt, row0, nbytes), "mlp_image_plan")
        key = tuple((nt[l], row0[l]) for l in range(L))
        hit = self._prepared.get(key)
        if hit is None:
            st = PsaMlp()
            C.memmove(C.byref(st), C.byref(self.struct), C.sizeof(PsaMlp))
            keep = []
            for l in range(L):
                if nbytes[l]:
                    w = self._weights[l]
                    img = torch.empty(int(nbytes[l]), dtype=torch.uint8, device=w.device)
                    check(lib.psa_prepare_weight_image(w.shape[0], w.shape[1], row0[l], nt[l], _ptr(w), _ptr(img), _stream()),
                          "prepare_weight_image")
                    st.image[l] = img.data_ptr(); st.image_nt[l] = nt[l]; st.image_row0[l] = row0[l]
                    keep.append(img)
            hit = (st, keep)
            self._prepared[key] = hit
        return C.byref(hit[0])


def shared_mlp(x: torch.Tensor, mlp: MlpParams, pool_k: int = 1) -> torch.Tensor:
    """Per-row shared MLP on dense rows: x (..., C_0) -> (..., C_L), or with pool_k > 1 the channel-wise max over
    every run of pool_k consecutive rows: (rows/pool_k, C_L)."""
    x = _dev(x, torch.float32, "x")
    c0 = x.shape[-1]
    if c0 != mlp.channels[0]:
        raise ValueError(f"shared_mlp: input width {c0} != {mlp.channels[0]}")
    rows = x.numel() // c0
    lead = x.shape[:-1]
    cl = mlp.channels[-1]
    lib = _lib.load()
    need = lib.psa_shared_mlp_workspace_bytes(rows, mlp.ref)
    ws = torch.empty((max(need, 4) + 3) // 4, dtype=torch.float32, device=x.device) if need else None
    if pool_k == 1:
        out = torch.empty((*lead, cl), dtype=torch.float32, device=x.device)
    else:
        out = torch.empty((rows // max(pool_k, 1), cl), dtype=torch.float32, device=x.device)
    check(lib.psa_shared_mlp(rows, pool_k, _ptr(x), mlp.prepared(0, rows, pool_k), _ptr(out), _ptr(ws), C.c_size_t(need), _stream()),
          "shared_mlp")
    return out


def shared_mlp_grouped(x: torch.Tensor, mlp: MlpParams, group_add: torch.Tensor) -> torch.Tensor:
    """shared_mlp whose first layer also adds one row of group_add (G, C_1) per group of rows/G consecutive rows before its
    affine: x (..., C_0) -> (..., C_L).  With the first weight split as [W_x; W_g], shared_mlp_grouped(x, mlp_x, g . W_g) is
    shared_mlp(concat([x, tile(g)]), mlp) without the concatenation (psa_shared_mlp_grouped)."""
    x = _dev(x, torch.float32, "x")
    group_add = _dev(group_add, torch.float32, "group_add", 2)
    c0 = x.shape[-1]
    if c0 != mlp.channels[0]:
        raise ValueError(f"shared_mlp_grouped: input width {c0} != {mlp.channels[0]}")
    rows = x.numel() // c0
    groups = group_add.shape[0]
    if group_add.shape[1] != mlp.channels[1]:
        raise ValueError(f"shared_mlp_grouped: group_add width {group_add.shape[1]} != {mlp.channels[1]}")
    if groups < 1 or rows % groups:
        raise ValueError(f"shared_mlp_grouped: {groups} groups do not divide {rows} rows")
    lib = _lib.load()
    need = lib.psa_shared_mlp_workspace_bytes(rows, mlp.ref)
    ws = torch.empty((max(need, 4) + 3) // 4, dtype=torch.float32, device=x.device) if need else None
    out = torch.empty((*x.shape[:-1], mlp.channels[-1]), dtype=torch.float32, device=x.device)
    check(lib.psa_shared_mlp_grouped(rows, rows // groups, _ptr(x), mlp.prepared(0, rows), _ptr(group_add), _ptr(out), _ptr(ws),
                                     C.c_size_t(need), _stream()), "shared_mlp_grouped")
    return out


def sa_module_infer(xyz, new_xyz, points, radius: float, nsample: int, mlp: MlpParams, idx=None, return_idx=False):
    """Fused set-abstraction level (inference): ball query + group + centre + MLP + max-pool.
    xyz (B,N,3), new_xyz (B,M,3), points (B,N,C) or None -> (B,M,C_L) [, idx (B,M,nsample), pts_cnt (B,M)]."""
    xyz = _dev(xyz, torch.float32, "xyz", 3)
    new_xyz = _dev(new_xyz, torch.float32, "new_xyz", 3)
    b, n, _ = xyz.shape
    m = new_xyz.shape[1]
    c = 0
    if points is not None:
        points = _dev(points, torch.float32, "points", 3)
        c = points.shape[2]
    out = torch.empty((b, m, mlp.channels[-1]), dtype=torch.float32, device=xyz.device)
    idx_out = cnt = None
    if idx is None:
        idx_out = torch.empty((b, m, nsample), dtype=torch.int32, device=xyz.device)
        cnt = torch.empty((b, m), dtype=torch.int32, device=xyz.device)
    else:
        idx = _dev(idx, torch.int32, "idx", 3)
    lib = _lib.load()
    need = lib.psa_sa_module_workspace_bytes(b, n, m, c, nsample, mlp.ref)
    ws = torch.empty((need + 3) // 4, dtype=torch.float32, device=xyz.device) if need else None   # torch allocations are 512-B aligned
    check(lib.psa_sa_module_infer(b, n, m, c, C.c_float(radius), nsample, _ptr(xyz), _ptr(new_xyz), _ptr(points),
                                  _ptr(idx), mlp.prepared(2, b * n, 1, c, nsample), _ptr(out), _ptr(idx_out), _ptr(cnt), _ptr(ws),
                                  C.c_size_t(need), _stream()), "sa_module_infer")
    if return_idx:
        return out, (idx if idx is not None else idx_out), cnt
    return out


def sa_group_all_infer(xyz, points, mlp: MlpParams) -> torch.Tensor:
    """pointnet_sa_module(group_all=True) fused: rows [xyz, points] -> MLP -> max over each cloud's points, no concat.
    xyz (B,N,3), points (B,N,C) -> (B, C_L).  Falls back to concat + shared_mlp when the shapes are not eligible."""
    xyz = _dev(xyz, torch.float32, "xyz", 3)
    points = _dev(points, torch.float32, "points", 3)
    b, n, _ = xyz.shape
    c = points.shape[2]
    lib = _lib.load()
    out = torch.empty((b, mlp.channels[-1]), dtype=torch.float32, device=xyz.device)
    need = lib.psa_sa_group_all_workspace_bytes(b, n, c, mlp.ref)
    ws = torch.empty((need + 3) // 4, dtype=torch.float32, device=xyz.device) if need else None
    rc = lib.psa_sa_group_all_infer(b, n, c, _ptr(xyz), _ptr(points), mlp.prepared(1, b * n, n, c), _ptr(out), _ptr(ws),
                                    C.c_size_t(need), _stream())
    if rc == -2:        # PSA_ERR_UNSUPPORTED: shapes outside the fused path
        rows = torch.cat([xyz, points], dim=2).reshape(b * n, 3 + c)
        return shared_mlp(rows, mlp, pool_k=n)
    check(rc, "sa_group_all_infer")
    return out


def sa_conv1_prebn(xyz, new_xyz, points, radius: float, nsample: int, w1, bias=None, want_stats: bool = True):
    """Training-mode front of a set-abstraction level (variant F1): ball query + group + centre + conv1 + bias in one
    launch.  -> pre (B,M,nsample,C1) PRE-batch-norm activations, idx (B,M,nsample), pts_cnt (B,M), stats (2,C1) =
    per-channel [sum, sum of squares] over all rows (None unless want_stats)."""
    xyz = _dev(xyz, torch.float32, "xyz", 3)
    new_xyz = _dev(new_xyz, torch.float32, "new_xyz", 3)
    w1 = _dev(w1, torch.float32, "w1", 2)
    b, n, _ = xyz.shape
    m = new_xyz.shape[1]
    c = 0
    if points is not None:
        points = _dev(points, torch.float32, "points", 3)
        c = points.shape[2]
    if w1.shape[0] != 3 + c:
        raise ValueError(f"sa_conv1_prebn: w1 has {w1.shape[0]} rows, expected 3 + {c}")
    c1 = w1.shape[1]
    if bias is not None:
        bias = _dev(bias, torch.float32, "bias", 1)
    dev = xyz.device
    pre = torch.empty((b, m, nsample, c1), dtype=torch.float32, device=dev)
    idx = torch.empty((b, m, nsample), dtype=torch.int32, device=dev)
    cnt = torch.empty((b, m), dtype=torch.int32, device=dev)
    stats = torch.empty((2, c1), dtype=torch.float32, device=dev) if want_stats else None
    lib = _lib.load()
    need = lib.psa_sa_conv1_prebn_workspace_bytes(b, n, m, c, c1, 1 if want_stats else 0)
    ws = torch.empty((need + 3) // 4, dtype=torch.float32, device=dev) if need else None
    check(lib.psa_sa_conv1_prebn(b, n, m, c, C.c_float(radius), nsample, _ptr(xyz), _ptr(new_xyz), _ptr(points), _ptr(w1),
                                 _ptr(bias), c1, _ptr(pre), _ptr(idx), _ptr(cnt), _ptr(stats), _ptr(ws), C.c_size_t(need),
                                 _stream()), "sa_conv1_prebn")
    return pre, idx, cnt, stats


def pool_rows(x, pool_k: int, mode: str = "max", dist=None) -> torch.Tensor:
    """x (G*pool_k, C) -> (G, C): 'max', 'avg' or 'weighted_avg' (weights exp(-5 d)/sum, dist (G*pool_k,)) over each run of
    pool_k rows -- the pooling modes of pointnet_sa_module (pointnet_util.py:126-146)."""
    x = _dev(x, torch.float32, "x", 2)
    rows, c = x.shape
    if rows % pool_k:
        raise ValueError(f"pool_rows: {rows} rows are not a multiple of pool_k={pool_k}")
    code = {"max": 0, "avg": 1, "weighted_avg": 2}[mode]
    if dist is not None:
        dist = _dev(dist.reshape(-1), torch.float32, "dist", 1)
    out = torch.empty((rows // pool_k, c), dtype=torch.float32, device=x.device)
    check(_lib.load().psa_pool_rows(rows // pool_k, pool_k, c, code, _ptr(x), _ptr(dist), _ptr(out), _stream()), "pool_rows")
    return out


def edgeconv_infer(x, nn_idx, mlp: MlpParams) -> torch.Tensor:
    """Fused EdgeConv (inference): x (B,N,C), nn_idx (B,N,k) -> (B,N,C_L) = max_j MLP([x_i, x_j - x_i])."""
    x = _dev(_squeeze_pc(x), torch.float32, "x", 3)
    nn_idx = _dev(nn_idx, torch.int32, "nn_idx", 3)
    b, n, c = x.shape
    k = nn_idx.shape[2]
    out = torch.empty((b, n, mlp.channels[-1]), dtype=torch.float32, device=x.device)
    lib = _lib.load()
    need = lib.psa_edgeconv_workspace_bytes(b, n, c, k, mlp.ref)
    ws = torch.empty((need + 3) // 4, dtype=torch.float32, device=x.device) if need else None
    check(lib.psa_edgeconv_infer(b, n, c, k, _ptr(x), _ptr(nn_idx), mlp.ref, _ptr(out), _ptr(ws), C.c_size_t(need), _stream()),
          "edgeconv_infer")
    return out


# ------------------------------------------------------------------------------------------------
# SpiderCNN
# ------------------------------------------------------------------------------------------------
def spider_conv(delta, nn_idx, feat, taylor, weights, bias, feat_scale=None, feat_shift=None) -> torch.Tensor:
    """One spiderConv layer up to its group norm, without the (B,N,k,C*T) product tensor (psa_spider_conv_infer):
    delta (B,N,k,3), nn_idx (B,N,k) int32, feat (B,N,C), taylor (20,T) (monomial order of include/psa.h), weights
    (1,k,C*T,C_out) or (k,C*T,C_out), bias (C_out) -> pre-group-norm y (B,N,C_out).  feat_scale / feat_shift (B,C): the
    previous layer's group norm, applied with a ReLU as feat is read; None: feat is read as it is."""
    delta = _dev(delta, torch.float32, "delta", 4)
    nn_idx = _dev(nn_idx, torch.int32, "nn_idx", 3)
    feat = _dev(feat, torch.float32, "feat", 3)
    taylor = _dev(taylor, torch.float32, "taylor", 2)
    weights = _dev(weights, torch.float32, "weights")
    bias = _dev(bias, torch.float32, "bias", 1)
    b, n, c = feat.shape
    k = nn_idx.shape[2]
    t = taylor.shape[1]
    c_out = bias.shape[0]
    if tuple(nn_idx.shape[:2]) != (b, n) or tuple(delta.shape) != (b, n, k, 3):
        raise ValueError(f"spider_conv: nn_idx {tuple(nn_idx.shape)} / delta {tuple(delta.shape)} do not match feat {tuple(feat.shape)}")
    if taylor.shape[0] != 20 or weights.numel() != k * c * t * c_out or weights.shape[-1] != c_out:
        raise ValueError(f"spider_conv: taylor {tuple(taylor.shape)} / weights {tuple(weights.shape)} do not match k={k} C={c} C_out={c_out}")
    if (feat_scale is None) != (feat_shift is None):
        raise ValueError("spider_conv: feat_scale and feat_shift go together")
    if feat_scale is not None:
        feat_scale = _dev(feat_scale, torch.float32, "feat_scale", 2)
        feat_shift = _dev(feat_shift, torch.float32, "feat_shift", 2)
        if tuple(feat_scale.shape) != (b, c) or tuple(feat_shift.shape) != (b, c):
            raise ValueError(f"spider_conv: feat_scale / feat_shift must be ({b}, {c})")
    y = torch.empty((b, n, c_out), dtype=torch.float32, device=feat.device)
    lib = _lib.load()
    need = lib.psa_spider_conv_workspace_bytes(b, n, c, k, t, c_out)
    ws = torch.empty((max(need, 4) + 3) // 4, dtype=torch.float32, device=feat.device)
    check(lib.psa_spider_conv_infer(b, n, c, k, t, c_out, _ptr(delta), _ptr(nn_idx), _ptr(feat), _ptr(feat_scale), _ptr(feat_shift),
                                    _ptr(taylor), _ptr(weights), _ptr(bias), _ptr(y), _ptr(ws), C.c_size_t(need), _stream()),
          "spider_conv")
    return y


def group_norm_affine(y, gamma, beta, groups: int, eps: float = 1e-6, apply: bool = False, relu: bool = False):
    """Group norm of y (B,N,C) over `groups` contiguous channel groups as a per-cloud affine (psa_group_norm_affine):
    -> (scale, shift) (B,C), or with apply=True (y * scale + shift [then ReLU], scale, shift)."""
    y = _dev(y, torch.float32, "y", 3)
    gamma = _dev(gamma, torch.float32, "gamma", 1)
    beta = _dev(beta, torch.float32, "beta", 1)
    b, n, c = y.shape
    if gamma.numel() != c or beta.numel() != c:
        raise ValueError(f"group_norm_affine: gamma / beta must have {c} entries")
    if groups < 1 or c % groups:
        raise ValueError(f"group_norm_affine: {groups} groups do not divide {c} channels")
    scale = torch.empty((b, c), dtype=torch.float32, device=y.device)
    shift = torch.empty((b, c), dtype=torch.float32, device=y.device)
    out = torch.empty_like(y) if apply else None
    check(_lib.load().psa_group_norm_affine(b, n, c, groups, C.c_float(eps), _ptr(y), _ptr(gamma), _ptr(beta), _ptr(scale), _ptr(shift),
                                            _ptr(out), 1 if relu else 0, _stream()), "group_norm_affine")
    return (out, scale, shift) if apply else (scale, shift)


def topk_pool(y, k: int = 2, scale=None, shift=None, relu: bool = False, out=None, offset: int = 0) -> torch.Tensor:
    """tf.nn.top_k over the points (SpiderCNN's topk_pool) of h = y [* scale + shift] [then ReLU]: y (B,N,C) -> (B,C,k), largest
    first.  out (B,C_total,k): written at channels [offset, offset + C) and returned."""
    y = _dev(y, torch.float32, "y", 3)
    b, n, c = y.shape
    if (scale is None) != (shift is None):
        raise ValueError("topk_pool: scale and shift go together")
    if scale is not None:
        scale = _dev(scale, torch.float32, "scale", 2)
        shift = _dev(shift, torch.float32, "shift", 2)
        if tuple(scale.shape) != (b, c) or tuple(shift.shape) != (b, c):
            raise ValueError(f"topk_pool: scale / shift must be ({b}, {c})")
    if out is None:
        out = torch.empty((b, c, k), dtype=torch.float32, device=y.device)
    elif not (out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.dim() == 3 and out.shape[0] == b and out.shape[2] == k):
        raise ValueError(f"topk_pool: out must be a contiguous float32 CUDA tensor ({b}, C_total, {k})")
    check(_lib.load().psa_topk_pool(b, n, c, k, _ptr(y), _ptr(scale), _ptr(shift), 1 if relu else 0, _ptr(out), out.shape[1], offset,
                                    _stream()), "topk_pool")
    return out


# --- SpiderCNN training backward (psa_spider_*: fp32 FMA, fixed-order sums) ---
def _spider_ws(b, n, c, k, t, c_out, device):
    need = int(_lib.load().psa_spider_conv_bwd_workspace_bytes(b, n, c, k, t, c_out))
    return torch.empty((max(need, 4) + 3) // 4, dtype=torch.float32, device=device), C.c_size_t(need)


def spider_taylor_filter(delta, taylor) -> torch.Tensor:
    """The Taylor filter values of spider_conv: delta (B,N,k,3), taylor (20,T) -> g (B,N,k,T)."""
    delta = _dev(delta, torch.float32, "delta", 4)
    taylor = _dev(taylor, torch.float32, "taylor", 2)
    b, n, k, three = delta.shape
    if three != 3 or taylor.shape[0] != 20:
        raise ValueError(f"spider_taylor_filter: delta {tuple(delta.shape)} / taylor {tuple(taylor.shape)}: want (B,N,k,3) / (20,T)")
    g = torch.empty((b, n, k, taylor.shape[1]), dtype=torch.float32, device=delta.device)
    check(_lib.load().psa_spider_taylor_filter(b, n, k, taylor.shape[1], _ptr(delta), _ptr(taylor), _ptr(g), _stream()), "spider_taylor_filter")
    return g


def _spider_bwd_inputs(nn_idx, feat, g, dy, feat_scale, feat_shift, what):
    nn_idx = _dev(nn_idx, torch.int32, "nn_idx", 3)
    feat = _dev(feat, torch.float32, "feat", 3)
    g = _dev(g, torch.float32, "g", 4)
    dy = _dev(dy, torch.float32, "dy", 3)
    b, n, c = feat.shape
    k = nn_idx.shape[2]
    if tuple(nn_idx.shape[:2]) != (b, n) or tuple(g.shape[:3]) != (b, n, k) or tuple(dy.shape[:2]) != (b, n):
        raise ValueError(f"{what}: nn_idx {tuple(nn_idx.shape)} / g {tuple(g.shape)} / dy {tuple(dy.shape)} do not match feat {tuple(feat.shape)}")
    if (feat_scale is None) != (feat_shift is None):
        raise ValueError(f"{what}: feat_scale and feat_shift go together")
    if feat_scale is not None:
        feat_scale = _dev(feat_scale, torch.float32, "feat_scale", 2)
        feat_shift = _dev(feat_shift, torch.float32, "feat_shift", 2)
        if tuple(feat_scale.shape) != (b, c) or tuple(feat_shift.shape) != (b, c):
            raise ValueError(f"{what}: feat_scale / feat_shift must be ({b}, {c})")
    return nn_idx, feat, g, dy, feat_scale, feat_shift


def spider_conv_bwd_weight(nn_idx, feat, g, dy, feat_scale=None, feat_shift=None) -> torch.Tensor:
    """The gradient of spider_conv's weights: nn_idx (B,N,k), feat (B,N,C), g (B,N,k,T) (spider_taylor_filter), dy (B,N,C_out) the
    gradient of y -> dW (k, C*T, C_out), the reference's row order (j, c, t)."""
    nn_idx, feat, g, dy, feat_scale, feat_shift = _spider_bwd_inputs(nn_idx, feat, g, dy, feat_scale, feat_shift, "spider_conv_bwd_weight")
    b, n, c = feat.shape
    k, t, c_out = nn_idx.shape[2], g.shape[3], dy.shape[2]
    dW = torch.empty((k, c * t, c_out), dtype=torch.float32, device=feat.device)
    ws, nbytes = _spider_ws(b, n, c, k, t, c_out, feat.device)
    check(_lib.load().psa_spider_conv_bwd_weight(b, n, c, k, t, c_out, _ptr(nn_idx), _ptr(feat), _ptr(feat_scale), _ptr(feat_shift), _ptr(g),
                                                 _ptr(dy), _ptr(dW), _ptr(ws), nbytes, _stream()), "spider_conv_bwd_weight")
    return dW


def spider_conv_bwd_data(nn_idx, feat, g, weights, dy, feat_scale=None, feat_shift=None, want_D: bool = True):
    """The data side of spider_conv's backward -> (D (B,N,k,C) or None, dg (B,N,k,T)): D[p,j,c] = sum_t g Q, dg[p,j,t] = sum_c h Q with
    Q[p,j,c,t] = sum_o dy[p,o] W[j,c*T+t,o].  group_point_grad(D, nn_idx) is the gradient of the layer's input activation."""
    nn_idx, feat, g, dy, feat_scale, feat_shift = _spider_bwd_inputs(nn_idx, feat, g, dy, feat_scale, feat_shift, "spider_conv_bwd_data")
    weights = _dev(weights, torch.float32, "weights")
    b, n, c = feat.shape
    k, t, c_out = nn_idx.shape[2], g.shape[3], dy.shape[2]
    if weights.numel() != k * c * t * c_out or weights.shape[-1] != c_out:
        raise ValueError(f"spider_conv_bwd_data: weights {tuple(weights.shape)} do not match k={k} C={c} T={t} C_out={c_out}")
    D = torch.empty((b, n, k, c), dtype=torch.float32, device=feat.device) if want_D else None
    dg = torch.empty((b, n, k, t), dtype=torch.float32, device=feat.device)
    check(_lib.load().psa_spider_conv_bwd_data(b, n, c, k, t, c_out, _ptr(nn_idx), _ptr(feat), _ptr(feat_scale), _ptr(feat_shift), _ptr(g),
                                               _ptr(weights), _ptr(dy), _ptr(D), _ptr(dg), _stream()), "spider_conv_bwd_data")
    return D, dg


def spider_taylor_grad(delta, dg) -> torch.Tensor:
    """The gradient of the (20,T) Taylor coefficients: delta (B,N,k,3), dg (B,N,k,T) -> (20,T), sums in fp64."""
    delta = _dev(delta, torch.float32, "delta", 4)
    dg = _dev(dg, torch.float32, "dg", 4)
    b, n, k, _ = delta.shape
    if delta.shape[3] != 3 or tuple(dg.shape[:3]) != (b, n, k):
        raise ValueError(f"spider_taylor_grad: delta {tuple(delta.shape)} / dg {tuple(dg.shape)} do not match")
    t = dg.shape[3]
    out = torch.empty((20, t), dtype=torch.float32, device=dg.device)
    ws, nbytes = _spider_ws(b, n, 1, k, t, 1, dg.device)
    check(_lib.load().psa_spider_taylor_grad(b, n, k, t, _ptr(delta), _ptr(dg), _ptr(out), t, _ptr(ws), nbytes, _stream()), "spider_taylor_grad")
    return out


def spider_gn_bwd(y, scale, shift, gamma, groups: int, dpool, offset: int = 0, dh_next=None, eps: float = 1e-6):
    """Backward of topk_pool(relu(group_norm(y))) plus a gradient dh_next (B,N,C) of the activation itself: y (B,N,C), scale / shift (B,C)
    (group_norm_affine), dpool (B,C_total,2) the pooled gradient whose channels [offset, offset + C) are this layer's ->
    (dy (B,N,C), dgamma (C), dbeta (C))."""
    y = _dev(y, torch.float32, "y", 3)
    scale = _dev(scale, torch.float32, "scale", 2)
    shift = _dev(shift, torch.float32, "shift", 2)
    gamma = _dev(gamma, torch.float32, "gamma", 1)
    dpool = _dev(dpool, torch.float32, "dpool", 3)
    b, n, c = y.shape
    if tuple(scale.shape) != (b, c) or tuple(shift.shape) != (b, c) or gamma.numel() != c:
        raise ValueError(f"spider_gn_bwd: scale / shift must be ({b}, {c}) and gamma ({c})")
    if dpool.shape[0] != b or dpool.shape[2] != 2 or not 0 <= offset <= dpool.shape[1] - c:
        raise ValueError(f"spider_gn_bwd: dpool {tuple(dpool.shape)} does not hold {c} channels at offset {offset}")
    if groups < 1 or c % groups:
        raise ValueError(f"spider_gn_bwd: {groups} groups do not divide {c} channels")
    if dh_next is not None:
        dh_next = _dev(dh_next, torch.float32, "dh_next", 3)
        if tuple(dh_next.shape) != (b, n, c):
            raise ValueError(f"spider_gn_bwd: dh_next must be ({b}, {n}, {c})")
    dy = torch.empty_like(y)
    dgamma = torch.empty(c, dtype=torch.float32, device=y.device)
    dbeta = torch.empty(c, dtype=torch.float32, device=y.device)
    ws = torch.empty(max(b * 2 * c * 2, 1), dtype=torch.float32, device=y.device)
    check(_lib.load().psa_spider_gn_bwd(b, n, c, groups, C.c_float(eps), _ptr(y), _ptr(scale), _ptr(shift), _ptr(gamma), _ptr(dpool),
                                        dpool.shape[1], offset, _ptr(dh_next), _ptr(dy), _ptr(dgamma), _ptr(dbeta), _ptr(ws),
                                        C.c_size_t(ws.numel() * 4), _stream()), "spider_gn_bwd")
    return dy, dgamma, dbeta


# ------------------------------------------------------------------------------------------------
# 3DmFV-Net
# ------------------------------------------------------------------------------------------------
def fisher_vector(points, w, mu, sigma) -> torch.Tensor:
    """get_3dmfv(flatten=False) before its final transpose (psa_fisher_vector): points (B,N,3), w (G), mu (G,3), sigma (G,3)
    standard deviations -> (B,G,20), power- and L2-normalised.  Computed in fp64 without any (B,N,G) tensor."""
    points = _dev(points, torch.float32, "points", 3)
    w = _dev(w, torch.float32, "w", 1)
    mu = _dev(mu, torch.float32, "mu", 2)
    sigma = _dev(sigma, torch.float32, "sigma", 2)
    b, n, d = points.shape
    g = w.shape[0]
    if d != 3 or tuple(mu.shape) != (g, 3) or tuple(sigma.shape) != (g, 3):
        raise ValueError(f"fisher_vector: points {tuple(points.shape)}, w {tuple(w.shape)}, mu {tuple(mu.shape)}, sigma "
                         f"{tuple(sigma.shape)}: expected (B,N,3), (G), (G,3), (G,3)")
    out = torch.empty((b, g, 20), dtype=torch.float32, device=points.device)
    check(_lib.load().psa_fisher_vector(b, n, g, _ptr(points), _ptr(w), _ptr(mu), _ptr(sigma), _ptr(out), _stream()), "fisher_vector")
    return out


def _rows_view(t: torch.Tensor, name: str) -> torch.Tensor:
    """a 2-D float32 CUDA tensor whose rows may be strided (a column slice of a wider buffer), or a contiguous copy"""
    if not isinstance(t, torch.Tensor) or t.dim() != 2:
        raise ValueError(f"{name}: expected a 2-D tensor (voxel rows, channels)")
    if t.stride(1) == 1 and t.stride(0) >= t.shape[1]:
        _dev(t[:0], torch.float32, name)          # device / dtype checks without a copy
        return t
    return _dev(t, torch.float32, name)


def conv3d(x, r: int, weights, scale, shift, relu: bool = True, out=None, offset: int = 0) -> torch.Tensor:
    """One tf_util.conv3d layer (SAME, stride 1) with folded batch norm on voxel-major rows (psa_conv3d_infer): x (B*r^3, C), row =
    voxel * B + cloud (a column slice of a wider buffer is read in place); weights (k,k,k,C,C_out) or (k^3*C, C_out) with k in
    {1, 3, 5}; scale (C_out) or None, shift (C_out) -> relu?((x * W) * scale + shift) (B*r^3, C_out).  out (B*r^3, C_total):
    written at channels [offset, offset + C_out) and returned."""
    x = _rows_view(x, "x")
    weights = _dev(weights, torch.float32, "weights")
    shift = _dev(shift, torch.float32, "shift", 1)
    rows, c = x.shape
    c_out = shift.shape[0]
    vox = r ** 3
    if r < 1 or rows % vox:
        raise ValueError(f"conv3d: {rows} rows are not a multiple of r^3 = {vox}")
    kk = weights.numel() // (c * c_out) if c * c_out else 0
    k = {1: 1, 27: 3, 125: 5}.get(kk)
    if k is None or weights.numel() != kk * c * c_out or weights.shape[-1] != c_out:
        raise ValueError(f"conv3d: weights {tuple(weights.shape)} are not (k,k,k,{c},{c_out}) with k in (1, 3, 5)")
    if weights.dim() == 5 and tuple(weights.shape) != (k, k, k, c, c_out):
        raise ValueError(f"conv3d: weights {tuple(weights.shape)} are not ({k},{k},{k},{c},{c_out})")
    if scale is not None:
        scale = _dev(scale, torch.float32, "scale", 1)
        if scale.shape[0] != c_out:
            raise ValueError(f"conv3d: scale must have {c_out} entries")
    if out is None:
        out = torch.empty((rows, c_out), dtype=torch.float32, device=x.device)
        view = out
    else:
        if not (out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.dim() == 2 and out.shape[0] == rows):
            raise ValueError(f"conv3d: out must be a contiguous float32 CUDA tensor ({rows}, C_total)")
        if offset < 0 or offset + c_out > out.shape[1]:
            raise ValueError(f"conv3d: channels [{offset}, {offset + c_out}) do not fit out's {out.shape[1]}")
        view = out[:, offset:]
    b = rows // vox
    lib = _lib.load()
    need = lib.psa_conv3d_workspace_bytes(b, r, k, c, c_out)
    ws = torch.empty((max(need, 4) + 3) // 4, dtype=torch.float32, device=x.device)
    check(lib.psa_conv3d_infer(b, r, k, c, c_out, _ptr(x), x.stride(0), _ptr(weights), _ptr(scale), _ptr(shift), 1 if relu else 0,
                               _ptr(view), out.stride(0), _ptr(ws), C.c_size_t(need), _stream()), "conv3d")
    return out


def _conv3d_bwd_ws(b, r, k, c, c_out, device) -> tuple[torch.Tensor, C.c_size_t]:
    need = int(_lib.load().psa_conv3d_bwd_workspace_bytes(b, r, k, c, c_out))
    return torch.empty((need + 3) // 4 + 64, dtype=torch.float32, device=device), C.c_size_t(need)


def _conv3d_k(kk: int) -> int:
    k = {1: 1, 27: 3, 125: 5}.get(kk)
    if k is None:
        raise ValueError(f"conv3d: {kk} taps, expected k^3 with k in (1, 3, 5)")
    return k


def conv3d_bwd_weight(x, r: int, dy, k: int) -> torch.Tensor:
    """The gradient of conv3d's weights (psa_conv3d_bwd_weight, fp32): x (B*r^3, C) voxel-major rows (a column slice is read in
    place), dy (B*r^3, C_out) the gradient of the conv's pre-batch-norm output -> dW (k,k,k,C,C_out), TF's kernel layout."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1):
        x = _dev(x, torch.float32, "x", 2)
    dy = _dev(dy, torch.float32, "dy", 2)
    rows, c = x.shape
    if rows % r ** 3 or dy.shape[0] != rows:
        raise ValueError(f"conv3d_bwd_weight: x has {rows} rows, dy {dy.shape[0]}; both must be B*r^3 with r = {r}")
    b, c_out = rows // r ** 3, dy.shape[1]
    dW = torch.empty((k, k, k, c, c_out), dtype=torch.float32, device=x.device)
    ws, wsn = _conv3d_bwd_ws(b, r, k, c, c_out, x.device)
    check(_lib.load().psa_conv3d_bwd_weight(b, r, k, c, c_out, _ptr(x), x.stride(0), _ptr(dy), _ptr(dW), _ptr(ws), wsn, _stream()),
          "conv3d_bwd_weight")
    return dW


def conv3d_bwd_data(dy, r: int, weights, out=None, accumulate: bool = False) -> torch.Tensor:
    """The gradient of conv3d's input (psa_conv3d_bwd_data, fp32): dy (B*r^3, C_out), weights (k,k,k,C,C_out) -> dx (B*r^3, C).
    out (B*r^3, >= C), possibly a column slice of a wider buffer: written in place, or added to with accumulate=True."""
    dy = _dev(dy, torch.float32, "dy", 2)
    weights = _dev(weights, torch.float32, "weights")
    rows, c_out = dy.shape
    c = weights.shape[-2] if weights.dim() == 5 else None
    if c is None or weights.shape[-1] != c_out or rows % r ** 3:
        raise ValueError(f"conv3d_bwd_data: weights {tuple(weights.shape)} are not (k,k,k,C,{c_out}), or {rows} rows are not B*r^3")
    k = _conv3d_k(weights.numel() // (c * c_out))
    if out is None:
        out = torch.empty((rows, c), dtype=torch.float32, device=dy.device)
    elif not (out.is_cuda and out.dtype == torch.float32 and out.dim() == 2 and out.shape[0] == rows and out.shape[1] >= c and out.stride(1) == 1):
        raise ValueError(f"conv3d_bwd_data: out must be a float32 CUDA tensor ({rows}, >= {c}) with unit column stride")
    b = rows // r ** 3
    ws, wsn = _conv3d_bwd_ws(b, r, k, c, c_out, dy.device)
    check(_lib.load().psa_conv3d_bwd_data(b, r, k, c, c_out, _ptr(dy), _ptr(weights), _ptr(out), out.stride(0), 1 if accumulate else 0,
                                          _ptr(ws), wsn, _stream()), "conv3d_bwd_data")
    return out


def conv3d_bwd_macs(b: int, r: int, k: int, c: int, c_out: int) -> tuple[int, int, int]:
    """(multiply-adds issued by the weight gradient, by the data gradient, multiply-adds with the tap inside the grid) at these dims"""
    v = [C.c_longlong(0) for _ in range(3)]
    check(_lib.load().psa_conv3d_bwd_macs(b, r, k, c, c_out, *(C.byref(t) for t in v)), "conv3d_bwd_macs")
    return tuple(int(t.value) for t in v)


def pool3d_max_train(x, r: int) -> tuple[torch.Tensor, torch.Tensor]:
    """pool3d(x, r, 'max') and its winners (psa_pool3d_max_train): -> (out, winner) (B*ceil(r/2)^3, C), winner uint8 = the first
    maximum's window position dz * 4 + dy * 2 + dx."""
    x = _dev(x, torch.float32, "x", 2)
    rows, c = x.shape
    if rows % r ** 3:
        raise ValueError(f"pool3d_max_train: {rows} rows are not a multiple of r^3 = {r ** 3}")
    b, ro = rows // r ** 3, (r + 1) // 2
    out = torch.empty((b * ro ** 3, c), dtype=torch.float32, device=x.device)
    win = torch.empty((b * ro ** 3, c), dtype=torch.uint8, device=x.device)
    check(_lib.load().psa_pool3d_max_train(b, r, c, _ptr(x), _ptr(out), _ptr(win), _stream()), "pool3d_max_train")
    return out, win


def pool3d_bwd(dout, r: int, kind: str, winner=None) -> torch.Tensor:
    """The backward of pool3d on an r^3 grid (psa_pool3d_bwd): 'avg' -> dx (B*r^3, C) from dout (B*r^3, C); 'max' -> dx from dout
    (B*ceil(r/2)^3, C) and pool3d_max_train's winners."""
    dout = _dev(dout, torch.float32, "dout", 2)
    if kind not in ("avg", "max"):
        raise ValueError(f"pool3d_bwd: kind must be 'avg' or 'max', got {kind!r}")
    ro = r if kind == "avg" else (r + 1) // 2
    rows, c = dout.shape
    if rows % ro ** 3:
        raise ValueError(f"pool3d_bwd: {rows} rows are not a multiple of {ro ** 3}")
    if kind == "max":
        if winner is None or winner.dtype != torch.uint8 or tuple(winner.shape) != tuple(dout.shape):
            raise ValueError("pool3d_bwd: 'max' needs pool3d_max_train's uint8 winners of dout's shape")
        winner = winner.contiguous()
    b = rows // ro ** 3
    dx = torch.empty((b * r ** 3, c), dtype=torch.float32, device=dout.device)
    check(_lib.load().psa_pool3d_bwd(b, r, c, 0 if kind == "avg" else 1, _ptr(dout), _ptr(winner if kind == "max" else None), _ptr(dx),
                                     _stream()), "pool3d_bwd")
    return dx


def pool3d(x, r: int, kind: str) -> torch.Tensor:
    """The inception module's pools on voxel-major rows x (B*r^3, C) (psa_pool3d): 'avg' = SAME 3^3 average, stride 1, over the
    in-grid cells -> (B*r^3, C); 'max' = SAME 2^3 max, stride 2 -> (B*ceil(r/2)^3, C)."""
    x = _dev(x, torch.float32, "x", 2)
    rows, c = x.shape
    if r < 1 or rows % r ** 3:
        raise ValueError(f"pool3d: {rows} rows are not a multiple of r^3 = {r ** 3}")
    if kind not in ("avg", "max"):
        raise ValueError(f"pool3d: kind must be 'avg' or 'max', got {kind!r}")
    b = rows // r ** 3
    ro = r if kind == "avg" else (r + 1) // 2
    out = torch.empty((b * ro ** 3, c), dtype=torch.float32, device=x.device)
    check(_lib.load().psa_pool3d(b, r, c, 0 if kind == "avg" else 1, _ptr(x), _ptr(out), _stream()), "pool3d")
    return out


# ------------------------------------------------------------------------------------------------
# PointCNN (PointCNN/pointcnn.py:10-52, pointfly.py:122-128, 163-176, 298-347)
# ------------------------------------------------------------------------------------------------
KNN_DILATED_MAX = 64          # k * d entries a query keeps (psa_knn_dilated)
XCONV_MAX_K = 16              # neighbours per query of psa_xconv_core
XCONV_WEIGHTS = ("w_pts0", "s_pts0", "t_pts0", "w_pts1", "s_pts1", "t_pts1", "w_x0", "s_x0", "t_x0", "w_x1", "s_x1", "t_x1", "w_x2",
                 "s_x2", "t_x2", "w_dw")


def knn_dilated(points, queries, k: int, d: int = 1) -> torch.Tensor:
    """knn_indices_general(queries, points, k*d, sort=True)[:, :, ::d] (psa_knn_dilated): points (B,N,3), queries (B,M,3) -> (B,M,k)
    int32 indices into points, ascending distance, lower index first on ties, duplicate points kept."""
    if k < 1 or d < 1 or k * d > KNN_DILATED_MAX:
        raise ValueError(f"knn_dilated: k={k}, d={d}: need k, d >= 1 and k*d <= {KNN_DILATED_MAX}")
    points = _dev(points, torch.float32, "points", 3)
    queries = _dev(queries, torch.float32, "queries", 3)
    b, n, c = points.shape
    if c != 3 or queries.shape[0] != b or queries.shape[2] != 3:
        raise ValueError(f"knn_dilated: points {tuple(points.shape)} / queries {tuple(queries.shape)} must be (B,N,3) / (B,M,3)")
    if k * d > n:
        raise ValueError(f"knn_dilated: k*d = {k * d} exceeds the {n} points")
    m = queries.shape[1]
    idx = torch.empty((b, m, k), dtype=torch.int32, device=points.device)
    check(_lib.load().psa_knn_dilated(b, n, m, k, d, _ptr(points), _ptr(queries), _ptr(idx), _stream()), "knn_dilated")
    return idx


def xconv_core(pts, qrs, idx, fts, weights: dict, dm: int) -> torch.Tensor:
    """One X-Conv layer up to the depthwise stage of its separable conv (psa_xconv_core): pts (B,N,3), qrs (B,P,3), idx (B,P,K) int32,
    fts (B,N,C_prev) or None; ``weights`` maps the names of ops.XCONV_WEIGHTS to the TF-shaped tensors (include/psa.h) -> (B*P,
    C_in*dm), C_in = C_pts + C_prev."""
    b, p, k = idx.shape
    w_pts0 = weights["w_pts0"]
    c_pts = w_pts0.shape[-1]
    c_prev = 0 if fts is None else fts.shape[-1]
    if k < 1 or k > XCONV_MAX_K:
        raise ValueError(f"xconv_core: K={k} must be in [1, {XCONV_MAX_K}]")
    if tuple(weights["w_x0"].shape[-3:]) != (k, 3, k * k) or tuple(weights["w_dw"].shape[-3:-1]) != (k, c_pts + c_prev):
        raise ValueError(f"xconv_core: X_0 {tuple(weights['w_x0'].shape)} / depthwise {tuple(weights['w_dw'].shape)} do not match K={k}, "
                         f"C_in={c_pts + c_prev}")
    if weights["w_dw"].shape[-1] != dm:
        raise ValueError(f"xconv_core: the depthwise kernel has multiplier {weights['w_dw'].shape[-1]}, not {dm}")
    pts = _dev(pts, torch.float32, "pts", 3)
    qrs = _dev(qrs, torch.float32, "qrs", 3)
    idx = _dev(idx, torch.int32, "idx", 3)
    if fts is not None:
        fts = _dev(fts, torch.float32, "fts", 3)
        if tuple(fts.shape[:2]) != tuple(pts.shape[:2]):
            raise ValueError(f"xconv_core: fts {tuple(fts.shape)} does not match pts {tuple(pts.shape)}")
    n = pts.shape[1]
    if qrs.shape[0] != b or qrs.shape[1] != p or pts.shape[0] != b:
        raise ValueError(f"xconv_core: pts {tuple(pts.shape)} / qrs {tuple(qrs.shape)} / idx {tuple(idx.shape)} disagree")
    ws = {name: _dev(weights[name], torch.float32, name) for name in XCONV_WEIGHTS}
    layer = _lib.PsaXconv(k, c_pts, c_prev, dm, *[ws[name].data_ptr() for name in XCONV_WEIGHTS])
    out = torch.empty((b * p, (c_pts + c_prev) * dm), dtype=torch.float32, device=pts.device)
    check(_lib.load().psa_xconv_core(b, n, p, _ptr(pts), _ptr(qrs), _ptr(idx), _ptr(fts), C.byref(layer), _ptr(out), _stream()),
          "xconv_core")
    return out


def dense_elu_affine(x, weights, scale, shift, bias=None, out=None, offset: int = 0) -> torch.Tensor:
    """elu(x . W [+ bias]) * scale + shift (psa_dense_elu_affine), PointCNN's dense / conv layer with ELU before its batch norm: x (R, K)
    (a column slice of a wider buffer is read in place), weights (K, N) or any TF shape (..., K, N) -> (R, N).  out (R, C_total):
    written at channels [offset, offset + N) and returned."""
    x = _rows_view(x, "x")
    weights = _dev(weights, torch.float32, "weights")
    rows, k = x.shape
    n = weights.shape[-1]
    if weights.numel() != k * n:
        raise ValueError(f"dense_elu_affine: weights {tuple(weights.shape)} are not ({k}, N)")
    scale = _dev(scale, torch.float32, "scale", 1)
    shift = _dev(shift, torch.float32, "shift", 1)
    if bias is not None:
        bias = _dev(bias, torch.float32, "bias", 1)
    for name, t in (("scale", scale), ("shift", shift), ("bias", bias)):
        if t is not None and t.shape[0] != n:
            raise ValueError(f"dense_elu_affine: {name} must have {n} entries")
    if out is None:
        out = torch.empty((rows, n), dtype=torch.float32, device=x.device)
        view = out
    else:
        if not (out.is_cuda and out.dtype == torch.float32 and out.dim() == 2 and out.stride(1) == 1 and out.shape[0] == rows):
            raise ValueError(f"dense_elu_affine: out must be a float32 CUDA tensor ({rows}, C_total) with unit column stride")
        if offset < 0 or offset + n > out.shape[1]:
            raise ValueError(f"dense_elu_affine: channels [{offset}, {offset + n}) do not fit out's {out.shape[1]}")
        view = out[:, offset:]
    lib = _lib.load()
    need = lib.psa_dense_elu_affine_workspace_bytes(rows, k, n)
    ws = torch.empty((max(need, 4) + 3) // 4, dtype=torch.float32, device=x.device)
    check(lib.psa_dense_elu_affine(rows, k, n, _ptr(x), x.stride(0), _ptr(weights), _ptr(bias), _ptr(scale), _ptr(shift), _ptr(view),
                                   out.stride(0), _ptr(ws), C.c_size_t(need), _stream()), "dense_elu_affine")
    return out


def set_mlp_mode(mode: int) -> None:
    """0 = tensor cores (wgmma) where the shapes allow, fp16x2 operands with the device-side range guard (default);
    1 = always the fp32-FMA kernels; 2 = tensor cores with bf16x3 operands (include/psa.h)."""
    check(_lib.load().psa_set_mlp_mode(int(mode)), "set_mlp_mode")


def get_mlp_mode() -> int:
    return int(_lib.load().psa_get_mlp_mode())




def elu_bn_dy(a, dh, ca, cb, cc, mask=None) -> torch.Tensor:
    """The gradient of z for a PointCNN layer BN(elu(z)) in training mode (psa_elu_bn_dy): a (R, C) = elu(z), the batch norm's input;
    dh (R, C) the gradient of its output (times mask, a dropout mask, when given); ca, cb, cc (C) the coefficients of
    psa_bn_bwd_coeffs -> (ca dh + cb a + cc) * (a < 0 ? a + 1 : 1), TF's EluGrad on the output."""
    a = _dev(a, torch.float32, "a", 2)
    dh = _dev(dh, torch.float32, "dh", 2)
    rows, c = a.shape
    if tuple(dh.shape) != (rows, c) or (mask is not None and tuple(mask.shape) != (rows, c)):
        raise ValueError(f"elu_bn_dy: dh {tuple(dh.shape)} and mask must match a {tuple(a.shape)}")
    ca, cb, cc = (_dev(t, torch.float32, n, 1) for t, n in ((ca, "ca"), (cb, "cb"), (cc, "cc")))
    if any(t.shape[0] != c for t in (ca, cb, cc)):
        raise ValueError(f"elu_bn_dy: ca, cb, cc must have {c} entries")
    mask = None if mask is None else _dev(mask, torch.float32, "mask", 2)
    g = _lib.PsaGradIn(y=_ptr(a), ld=c, ca=_ptr(ca), cb=_ptr(cb), cc=_ptr(cc), dh=_ptr(dh), ld_dh=c, mask=_ptr(mask), pool_k=1, C=c)
    dz = torch.empty_like(a)
    check(_lib.load().psa_elu_bn_dy(rows, c, C.byref(g), _ptr(dz), _stream()), "elu_bn_dy")
    return dz


def bn_affine_rows(a, scale, shift, out=None, offset: int = 0) -> torch.Tensor:
    """a * scale + shift per channel (psa_bn_affine_rows): a (R, C) -> (R, C), or written at channels [offset, offset + C) of out
    (R, C_total) and out returned."""
    a = _dev(a, torch.float32, "a", 2)
    rows, c = a.shape
    scale = _dev(scale, torch.float32, "scale", 1)
    shift = _dev(shift, torch.float32, "shift", 1)
    if scale.shape[0] != c or shift.shape[0] != c:
        raise ValueError(f"bn_affine_rows: scale and shift must have {c} entries")
    if out is None:
        out = torch.empty_like(a)
    elif not (out.is_cuda and out.dtype == torch.float32 and out.dim() == 2 and out.stride(1) == 1 and out.shape[0] == rows
              and 0 <= offset and offset + c <= out.shape[1]):
        raise ValueError(f"bn_affine_rows: out must be a float32 CUDA tensor ({rows}, >= {offset + c}) with unit column stride")
    check(_lib.load().psa_bn_affine_rows(rows, c, _ptr(a), _ptr(scale), _ptr(shift), C.c_void_p(out.data_ptr() + 4 * offset), out.stride(0),
                                         _stream()), "bn_affine_rows")
    return out


def xconv_depthwise_bwd(x, scale, shift, a, dh, ca, cb, cc, weights, elu: bool):
    """Backward of PointCNN's depthwise X layer z = depthwise(x * scale + shift, W) followed by BN(elu(z)) (elu=True, X_1) or BN(z)
    (X_2) in training mode (psa_xconv_depthwise_bwd): x, a (R, K*K) the saved activations of the input layer and of this one, dh
    (R, K*K) the gradient of this layer's batch-norm output, ca, cb, cc its psa_bn_bwd_coeffs, weights (..., K, K, K) -> (dW (K, K, K),
    dx (R, K*K) the gradient of x * scale + shift)."""
    x = _dev(x, torch.float32, "x", 2)
    a = _dev(a, torch.float32, "a", 2)
    dh = _dev(dh, torch.float32, "dh", 2)
    rows, kk = x.shape
    k = int(round(kk ** 0.5))
    if k * k != kk or not 1 <= k <= XCONV_MAX_K or tuple(a.shape) != (rows, kk) or tuple(dh.shape) != (rows, kk):
        raise ValueError(f"xconv_depthwise_bwd: x {tuple(x.shape)}, a {tuple(a.shape)}, dh {tuple(dh.shape)} must be (R, K*K), K <= {XCONV_MAX_K}")
    weights = _dev(weights, torch.float32, "weights")
    if tuple(weights.shape[-3:]) != (k, k, k):
        raise ValueError(f"xconv_depthwise_bwd: weights {tuple(weights.shape)} are not (..., {k}, {k}, {k})")
    vec = [_dev(t, torch.float32, n, 1) for t, n in ((scale, "scale"), (shift, "shift"), (ca, "ca"), (cb, "cb"), (cc, "cc"))]
    if any(t.shape[0] != kk for t in vec):
        raise ValueError(f"xconv_depthwise_bwd: scale, shift, ca, cb, cc must have {kk} entries")
    scale, shift, ca, cb, cc = vec
    lib = _lib.load()
    g = _lib.PsaGradIn(y=_ptr(a), ld=kk, ca=_ptr(ca), cb=_ptr(cb), cc=_ptr(cc), dh=_ptr(dh), ld_dh=kk, pool_k=1, C=kk)
    need = int(lib.psa_xconv_train_bwd_workspace_bytes(rows, 1, k, 1, 0, 1))
    ws = torch.empty(max(need, 4) // 4, dtype=torch.float32, device=x.device)
    dW = torch.empty((k, k, k), dtype=torch.float32, device=x.device)
    dx = torch.empty_like(x)
    check(lib.psa_xconv_depthwise_bwd(rows, k, _ptr(x), _ptr(scale), _ptr(shift), C.byref(g), int(bool(elu)), _ptr(weights), _ptr(dW), _ptr(dx),
                                      _ptr(ws), C.c_size_t(need), _stream()), "xconv_depthwise_bwd")
    return dW, dx
