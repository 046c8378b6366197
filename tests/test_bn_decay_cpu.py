"""The moving-average decay that training mode uses when no bn_decay is passed, and dgcnn_bga's joint loss, on the CPU."""
from types import SimpleNamespace

import numpy as np
import torch

from scanobjectnn_b200 import dgcnn, training


def _stub(frozen):
    return SimpleNamespace(frozen=frozen, fp=SimpleNamespace(flat=torch.zeros(8)))


def test_bn_decay_none_is_the_references_0_9():
    """every reference tf_util resolves bn_decay=None to 0.9 (`decay = bn_decay if bn_decay is not None else 0.9`)"""
    tr = _stub(False)
    flat, decay = training._flat_and_decay(tr, None)
    assert decay == 0.9 and flat is tr.fp.flat and flat.requires_grad
    assert training._flat_and_decay(_stub(False), 0.5)[1] == 0.5
    assert training._flat_and_decay(_stub(False), 0.99)[1] == 0.99
    assert training._flat_and_decay(_stub(True), None) == (None, 0.0)          # a frozen trainer neither updates nor differentiates


def test_dgcnn_bga_loss_matches_float64():
    """dgcnn.get_loss_bga against float64 written out: (1 - w) * mean CE of the classes + w * mean over clouds of the mean per-point
    2-way CE (dgcnn_bga.py:137-152), without dgcnn.get_loss's label smoothing; logits far from zero so no term is negligible"""
    rng = np.random.default_rng(3)
    b, n, c = 5, 37, 15
    cp = rng.normal(0, 4, (b, c)) + 20.0
    sp = rng.normal(0, 4, (b, n, 2))
    label, mask = rng.integers(0, c, b), rng.integers(0, 2, (b, n))

    def ce(logits, lab):
        z = logits - logits.max(-1, keepdims=True)
        lse = np.log(np.exp(z).sum(-1))
        return lse - np.take_along_axis(z, lab[..., None], -1)[..., 0]

    cls64 = ce(cp, label).mean()
    seg64 = ce(sp, mask).mean(1).mean()
    t = lambda a: torch.tensor(a, dtype=torch.float32)          # noqa: E731
    for w in (0.5, 0.2):
        total, cls, seg = dgcnn.get_loss_bga(t(cp), t(sp), torch.tensor(label), torch.tensor(mask, dtype=torch.int32), seg_weight=w)
        for got, want in ((cls, cls64), (seg, seg64), (total, (1 - w) * cls64 + w * seg64)):
            assert abs(float(got) - want) <= 1e-6 * max(1.0, abs(want)), (w, float(got), want)
    smoothed = float(dgcnn.get_loss(t(cp), torch.tensor(label)))
    assert abs(smoothed - cls64) > 1e-2, "dgcnn_bga's classification loss has no label smoothing"
