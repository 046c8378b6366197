"""The moving averages of every training model when get_model(is_training=True) gets no bn_decay: they must move as with the reference's
default 0.9, bit for bit, and differ from a run at 0.5 in every batch-normed layer.  dgcnn_bga's seg/conv1 and seg/conv2 are built
without bn_decay in the reference (dgcnn_bga.py:125-128), so they decay at 0.9 whatever the model's bn_decay."""
import pytest
import torch

from scanobjectnn_b200 import dgcnn, pointnet2_cls_bga, pointnet2_cls_partseg, pointnet2_cls_ssg, pointnet_cls, pointnet_partseg, pointnet_seg
from scanobjectnn_b200.synthetic import make_clouds

from . import gpu_util as G
from .restate import moving

pytestmark = pytest.mark.gpu
B, N = 8, 1024
SEG_DEFAULT = ("seg/conv1/", "seg/conv2/")         # dgcnn_bga's layers without bn_decay

MODELS = {
    "pointnet2_cls_ssg": (pointnet2_cls_ssg.init_params, pointnet2_cls_ssg.get_model),
    "pointnet2_cls_bga": (pointnet2_cls_bga.init_params, pointnet2_cls_bga.get_model),
    "pointnet2_cls_partseg": (pointnet2_cls_partseg.init_params, pointnet2_cls_partseg.get_model),
    "pointnet_cls": (pointnet_cls.init_params, pointnet_cls.get_model),
    "pointnet_seg": (pointnet_seg.init_params, pointnet_seg.get_model),
    "pointnet_partseg": (pointnet_partseg.init_params, pointnet_partseg.get_model),
    "dgcnn": (dgcnn.init_params, dgcnn.get_model),
    "dgcnn_bga": (lambda **kw: dgcnn.init_params(bga=True, **kw), dgcnn.get_model_bga),
}


def _moving_after_one_step(name, **decay):
    """the moving averages after and before one training-mode forward of a fresh store (same seed, same dropout draws) with `decay`
    passed on"""
    init, get_model = MODELS[name]
    p = init(seed=4, randomize_bn=True)
    before = moving(p)
    x = G.cu(make_clouds("ball", B, N, seed=104))
    torch.manual_seed(0)
    with torch.no_grad():
        get_model(x, True, params=p, **decay)
    torch.cuda.synchronize()
    return moving(p), before


@pytest.mark.parametrize("name", sorted(MODELS))
def test_bn_decay_none_moves_the_averages_as_0_9(name):
    default, before = _moving_after_one_step(name)
    at_09, _ = _moving_after_one_step(name, bn_decay=0.9)
    at_05, _ = _moving_after_one_step(name, bn_decay=0.5)
    assert default.keys() == at_09.keys() == before.keys() and default
    differ = [k for k in default if not torch.equal(default[k], at_09[k])]
    assert not differ, f"bn_decay=None does not move these moving averages as 0.9 does: {differ}"
    unmoved = [k for k in default if torch.equal(default[k], before[k])]
    assert not unmoved, f"not updated by a training step: {unmoved}"
    fixed = {k for k in at_05 if name == "dgcnn_bga" and k.startswith(SEG_DEFAULT)}
    same = [k for k in at_05 if k not in fixed and torch.equal(at_05[k], at_09[k])]
    assert not same, f"bn_decay=0.5 moves these moving averages as 0.9 does: {same}"
    if name == "dgcnn_bga":
        assert len(fixed) == 4
        moved = [k for k in fixed if not torch.equal(at_05[k], at_09[k])]
        assert not moved, f"the reference decays these at 0.9 whatever bn_decay is: {moved}"
