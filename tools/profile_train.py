"""One training step of pointnet2_cls_ssg at the bench shape (B=32, N=2048), for ncu launch lists:
  ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file train_launches.csv python tools/profile_train.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from scanobjectnn_b200 import pointnet2_cls_ssg
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.training import PointNet2ClsTrainer

B, N = 32, 2048
p = pointnet2_cls_ssg.init_params(seed=1)
tr = PointNet2ClsTrainer(p, B, N, 15)
x = torch.from_numpy(make_clouds("ball", B, N, seed=1001)).cuda()
y = torch.from_numpy(np.arange(B, dtype=np.int32) % 15).cuda()
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 1
for _ in range(steps):
    loss = tr.train_step(x, y)
torch.cuda.synchronize()
print("loss", float(loss.item()))
