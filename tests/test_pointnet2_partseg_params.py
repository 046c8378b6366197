"""pointnet2_cls_partseg's variables (CPU): the reference's names and shapes (pointnet2/models/pointnet2_cls_partseg.py:29-43, with
tf_util.conv2d kernels (1,1,Cin,Cout), tf_util.conv1d kernels (1,Cin,Cout) and batch norm under <scope>/bn), and a TF checkpoint
round trip through the store."""
import numpy as np
import pytest

from scanobjectnn_b200 import checkpoint as ck
from scanobjectnn_b200 import pointnet2_cls_partseg

CONV = {"layer1/conv0": (3, 64), "layer1/conv1": (64, 64), "layer1/conv2": (64, 128),
        "layer2/conv0": (131, 128), "layer2/conv1": (128, 128), "layer2/conv2": (128, 256),
        "layer3/conv0": (259, 256), "layer3/conv1": (256, 512), "layer3/conv2": (512, 1024),
        "fa_layer1/conv_0": (1280, 256), "fa_layer1/conv_1": (256, 256),
        "fa_layer2/conv_0": (384, 256), "fa_layer2/conv_1": (256, 128),
        "fa_layer3/conv_0": (128, 128), "fa_layer3/conv_1": (128, 128), "fa_layer3/conv_2": (128, 128)}


def _reference_shapes(num_class):
    want = {}
    for scope, (cin, cout) in CONV.items():
        want[f"{scope}/weights"] = (1, 1, cin, cout)
        want[f"{scope}/biases"] = (cout,)
        for v in ("beta", "gamma", "moving_mean", "moving_variance"):
            want[f"{scope}/bn/{v}"] = (cout,)
    want.update({"seg_fc1/weights": (1, 128, 128), "seg_fc1/biases": (128,), "seg_fc2/weights": (1, 128, num_class), "seg_fc2/biases": (num_class,)})
    for v in ("beta", "gamma", "moving_mean", "moving_variance"):
        want[f"seg_fc1/bn/{v}"] = (128,)
    return want


@pytest.mark.parametrize("num_class", [6, 3])
def test_init_params_has_the_reference_variables(num_class):
    p = pointnet2_cls_partseg.init_params(num_class, device="cpu")
    assert {k: tuple(v.shape) for k, v in p.items()} == _reference_shapes(num_class)


def test_store_survives_a_tf_checkpoint_round_trip(tmp_path):
    p = pointnet2_cls_partseg.init_params(seed=2, device="cpu", randomize_bn=True)
    src = {k: v.numpy().copy() for k, v in p.items()}
    prefix = str(tmp_path / "model.ckpt")
    ck.write_tf_checkpoint(prefix, src)
    q = pointnet2_cls_partseg.init_params(seed=7, device="cpu")
    assert ck.restore(q, prefix) == []
    for k in p:
        assert q[k].shape == p[k].shape and np.array_equal(q[k].numpy(), src[k]), k


def test_num_class_must_agree_with_the_store():
    p = pointnet2_cls_partseg.init_params(4, device="cpu")
    with pytest.raises(ValueError, match="num_class=6"):
        pointnet2_cls_partseg.get_model(np.zeros((1, 8, 3), np.float32), False, params=p)
