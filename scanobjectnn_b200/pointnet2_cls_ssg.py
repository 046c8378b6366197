"""pointnet2/models/pointnet2_cls_ssg.py on the libpsa kernels: get_model(point_cloud, is_training, bn_decay,
num_class) -> (logits (B,num_class), end_points), same layer hyper-parameters (pointnet2_cls_ssg.py:35-45)."""
from __future__ import annotations

import torch

from . import ops
from .pointnet_util import add_sa_module_params, pointnet_sa_module
from .tf_util import VariableStore, _require_inference

NUM_CLASSES = 15
_SIDE = {}


def _side_stream(device):
    key = torch.device(device).index if torch.device(device).index is not None else torch.cuda.current_device()
    if key not in _SIDE:
        _SIDE[key] = torch.cuda.Stream(device=key)
    return _SIDE[key]


def init_params(num_class=NUM_CLASSES, seed=0, device="cuda", randomize_bn=False) -> VariableStore:
    p = VariableStore(device=device, seed=seed)
    add_sa_module_params(p, "layer1", 3, [64, 64, 128], randomize_bn=randomize_bn)
    add_sa_module_params(p, "layer2", 3 + 128, [128, 128, 256], randomize_bn=randomize_bn)
    add_sa_module_params(p, "layer3", 3 + 256, [256, 512, 1024], randomize_bn=randomize_bn)
    p.add_fc("fc1", 1024, 512, bn=True, randomize_bn=randomize_bn)
    p.add_fc("fc2", 512, 256, bn=True, randomize_bn=randomize_bn)
    p.add_fc("fc3", 256, num_class, bn=False)
    return p


def get_model(point_cloud, is_training, bn_decay=None, num_class=NUM_CLASSES, *, params: VariableStore):
    """Classification PointNet++ (SSG): input (B,N,3), output (B,num_class).

    is_training=True: batch-statistics batch norm in every layer (moving averages updated with ``bn_decay``), dropout in
    the head, and logits that carry a grad_fn -- ``get_loss(...).backward()`` runs the hand-written backward kernels and
    leaves the gradient of every variable in ``params._flat.grad_of(name)`` (training.py)."""
    from .training import get_model_training, wants_input_grad
    frozen = not is_training and wants_input_grad(point_cloud)
    if is_training or frozen:
        # frozen: inference mode with a gradient w.r.t. the point cloud (batch norm on the moving averages, no dropout, the training
        # kernels); calls that need no gradient stay on the fused inference kernels below
        logits, tr = get_model_training(point_cloud, bn_decay, num_class, params, frozen=frozen)
        lv = tr.levels
        end_points = {"l0_xyz": point_cloud, "l1_xyz": lv[0].new_xyz, "l1_points": lv[0].pooled.view(point_cloud.shape[0], lv[0].m, -1),
                      "l1_indices": lv[0].idx, "l2_xyz": lv[1].new_xyz, "l2_points": lv[1].pooled.view(point_cloud.shape[0], lv[1].m, -1),
                      "l2_indices": lv[1].idx, "l3_points": lv[2].pooled.view(point_cloud.shape[0], 1, -1)}
        return logits, end_points
    batch_size = point_cloud.shape[0]
    end_points = {"l0_xyz": point_cloud}
    l0_xyz, l0_points = point_cloud, None
    # Sampling of BOTH levels up front: level 2's FPS needs level 1's centroids only, so it runs on a side stream while
    # the main stream does level 1's ball query + MLP (the FPS kernels occupy one CTA per cloud: 32 of 132 SMs).
    _, l1_new = ops.farthest_point_sample_and_gather(512, l0_xyz)
    main = torch.cuda.current_stream()
    side = _side_stream(point_cloud.device)
    fork = torch.cuda.Event()
    fork.record(main)
    side.wait_event(fork)
    with torch.cuda.stream(side):
        _, l2_new = ops.farthest_point_sample_and_gather(128, l1_new)
        join = torch.cuda.Event()
        join.record(side)
    l1_xyz, l1_points, l1_indices = pointnet_sa_module(l0_xyz, l0_points, npoint=512, radius=0.2, nsample=32,
                                                       mlp=[64, 64, 128], mlp2=None, group_all=False,
                                                       is_training=is_training, bn_decay=bn_decay, scope="layer1",
                                                       use_nchw=True, params=params, new_xyz=l1_new)
    main.wait_event(join)
    l2_new.record_stream(main)
    l2_xyz, l2_points, l2_indices = pointnet_sa_module(l1_xyz, l1_points, npoint=128, radius=0.4, nsample=64,
                                                       mlp=[128, 128, 256], mlp2=None, group_all=False,
                                                       is_training=is_training, bn_decay=bn_decay, scope="layer2",
                                                       params=params, new_xyz=l2_new)
    l3_xyz, l3_points, l3_indices = pointnet_sa_module(l2_xyz, l2_points, npoint=None, radius=None, nsample=None,
                                                       mlp=[256, 512, 1024], mlp2=None, group_all=True,
                                                       is_training=is_training, bn_decay=bn_decay, scope="layer3",
                                                       params=params)
    net = l3_points.reshape(batch_size, -1)
    # fc1 -> dp1 -> fc2 -> dp2 -> fc3 (dropout is the identity at inference): one 3-layer shared MLP
    head = params.mlp(["fc1", "fc2", "fc3"], [True, True, False])
    net = ops.shared_mlp(net, head)
    end_points.update(l1_xyz=l1_xyz, l1_points=l1_points, l1_indices=l1_indices, l2_xyz=l2_xyz, l2_points=l2_points,
                      l2_indices=l2_indices, l3_points=l3_points)
    return net, end_points


def get_loss(pred, label, end_points=None):
    """mean sparse softmax cross-entropy (pointnet2_cls_ssg.py:50-57)."""
    return torch.nn.functional.cross_entropy(pred, label.long())
