"""pointnet/models/pointnet_partseg.py: PointNet part segmentation (train_partseg.py), pointnet_cls's trunk and pointnet_seg's head
without the classification branch.  get_model(point_cloud, is_training, bn_decay, num_class) -> (seg_pred (B,N,num_class),
end_points), in inference, training and inference differentiable in the point cloud, as pointnet_seg.get_model.  The number of
parts is that of the store (init_params(num_class)); get_model's num_class is the reference's argument and must agree."""
from __future__ import annotations

from . import pointnet_cls
from .pointnet_seg import add_seg_head_params, seg_cross_entropy, seg_head, seg_head_training, transform_regulariser
from .tf_util import VariableStore

NUM_CLASSES = 6


def init_params(num_class=NUM_CLASSES, seed=0, device="cuda", randomize_bn=False) -> VariableStore:
    p = VariableStore(device=device, seed=seed)
    pointnet_cls.add_trunk_params(p, randomize_bn)
    add_seg_head_params(p, num_class, randomize_bn)
    return p


def get_model(point_cloud, is_training, bn_decay=None, num_class=NUM_CLASSES, *, params: VariableStore):
    from .training import wants_input_grad
    if params["conv10/weights"].shape[-1] != num_class:
        raise ValueError(f"num_class={num_class}, but the store's conv10 has {params['conv10/weights'].shape[-1]} outputs")
    frozen = not is_training and wants_input_grad(point_cloud)
    if is_training or frozen:
        point_feat, global_feat, end_points = pointnet_cls.trunk_training(point_cloud, bn_decay, params, frozen)
        return seg_head_training(point_feat, global_feat, bn_decay, params, frozen), end_points
    point_feat, global_feat, end_points = pointnet_cls.trunk(point_cloud, params)
    return seg_head(point_feat, global_feat, params), end_points


def get_loss(seg_pred, gt_seg, end_points, reg_weight=0.001):
    """pointnet_partseg.py:96-124: per-cloud mean point cross-entropy, averaged, + reg_weight l2_loss(T T^t - I)."""
    return seg_cross_entropy(seg_pred, gt_seg) + reg_weight * transform_regulariser(end_points)
