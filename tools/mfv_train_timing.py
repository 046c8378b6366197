"""3DmFV-Net training at N=1024, B=64 (train.py's default) and B=32: the conv3d backward of csrc/mfv_train.cu
(mfv_net_cls.get_model_training) against a torch autograd composition, tools/mfv_timing.py's Composed with batch statistics
(F.conv3d, F.batch_norm in training mode, fp32, TF32 off).

  per layer   every conv3d: forward + backward of one layer (conv, batch statistics, ReLU, and the gradients of its variables and of
              its input), GPU time between CUDA events, the two paths alternated window by window, median of the windows
  whole step  get_model_training + cross-entropy + backward in clouds/s; the composition runs the same Fisher vector and the same
              head (training.mlp_training) around its composed conv stack
  memory      the rise of torch.cuda.max_memory_allocated over one step of each
  MACs        per conv, the multiply-adds each gradient product issues against those whose tap lies inside the grid

Prints the card's name and power limit, then one JSON line.  Usage: python tools/mfv_train_timing.py [--batch 64 32] [--windows 10]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.nn.functional as F

from scanobjectnn_b200 import mfv_net_cls as M
from scanobjectnn_b200 import ops
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import BN_EPS
from scanobjectnn_b200.training import mlp_training

N = 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def window_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def alternate(fa, fb, windows, reps):
    """median ms per call of fa and fb, alternated window by window after one warm-up window each"""
    window_ms(fa, reps), window_ms(fb, reps)
    ta, tb = [], []
    for _ in range(windows):
        ta.append(window_ms(fa, reps))
        tb.append(window_ms(fb, reps))
    return float(np.median(ta)), float(np.median(tb))


def peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


class ComposedTrain:
    """the conv stack as torch autograd ops with batch statistics (tools/mfv_timing.py's Composed in training mode)"""

    def __init__(self, p):
        self.p = p
        self.v = {}
        for scope, k, cin, cout in M._module_widths():
            self.v[scope] = [p[f"{scope}/weights"].permute(4, 3, 0, 1, 2).contiguous().requires_grad_(True),
                             p[f"{scope}/biases"].clone().requires_grad_(True), p[f"{scope}/bn/gamma"].clone().requires_grad_(True),
                             p[f"{scope}/bn/beta"].clone().requires_grad_(True), p[f"{scope}/bn/moving_mean"].clone(),
                             p[f"{scope}/bn/moving_variance"].clone()]

    def conv(self, x, scope):
        W, b, g, be, mm, mv = self.v[scope]
        y = F.conv3d(x, W, b, padding=W.shape[-1] // 2)
        return torch.relu(F.batch_norm(y, mm, mv, g, be, training=True, momentum=0.1, eps=BN_EPS))

    def inception(self, x, scope):
        one = self.conv(x, f"{scope}_conv1")
        avg = F.avg_pool3d(x, 3, stride=1, padding=1, count_include_pad=False)
        return torch.cat([one, self.conv(one, f"{scope}_conv2"), self.conv(one, f"{scope}_conv3"), self.conv(avg, f"{scope}_conv4")], 1)

    def logits(self, points, gmm):
        fv = ops.fisher_vector(points, *gmm)
        b, g, _ = fv.shape
        r = round(g ** (1 / 3))
        net = fv.permute(0, 2, 1).reshape(b, 20, r, r, r)
        for l in (1, 2, 3):
            net = self.inception(net, f"inception{l}")
        net = F.max_pool3d(net, 2, 2, ceil_mode=True)
        for l in (4, 5):
            net = self.inception(net, f"inception{l}")
        net = F.max_pool3d(net, 2, 2, ceil_mode=True)
        net = net.permute(0, 2, 3, 4, 1).reshape(b, -1)
        for scope in ("fc1", "fc2", "fc3"):
            net = F.dropout(mlp_training(net, [(scope, True)], None, self.p), 0.3, training=True)
        return mlp_training(net, [("fc4", False)], None, self.p)


def layer_cases(tr, comp, b):
    """per conv: (name, fused fwd+bwd, composed fwd+bwd, (k, c, cout, r))"""
    out = []
    for li, m in enumerate(tr.modules):
        r, n, cin = m["r"], m["n"], m["cin"]
        for j, cv in enumerate(m["convs"]):
            src, ld = (m["X"], cin) if j == 0 else (m["H"], 3 * n) if j < 3 else (m["P"], cin)
            dx = None if li == 0 and j in (0, 3) else (m["dH"] if j in (1, 2) else m["dx4"])
            ldx = 3 * n if j in (1, 2) else cin

            def fused(m=m, cv=cv, src=src, ld=ld, dx=dx, ldx=ldx):
                tr._conv_fwd(m, cv, src, ld, 0.9)
                tr._conv_bwd(m, cv, src, ld, dx, ldx, False)

            scope = cv["scope"]
            x = torch.relu(torch.randn((b, cv["c"], r, r, r), device="cuda")).requires_grad_(li > 0 or j in (1, 2))
            gy = torch.randn((b, cv["cout"], r, r, r), device="cuda")

            def composed(x=x, gy=gy, scope=scope):
                comp.conv(x, scope).backward(gy)

            out.append((scope, fused, composed, (cv["k"], cv["c"], cv["cout"], r)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[64, 32])
    ap.add_argument("--windows", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    print(f"# {card()}; GPU time between CUDA events, fused and composed alternated window by window ({a.reps} calls per window), "
          f"median of {a.windows} windows after one warm-up window")
    gmm = [torch.from_numpy(t).cuda() for t in M.get_3d_grid_gmm((5, 5, 5))]
    result = {"card": card(), "n": N, "batches": {}}
    for b in a.batch:
        p = M.init_params(seed=1, randomize_bn=True)
        pc = M.init_params(seed=1, randomize_bn=True)
        comp = ComposedTrain(pc)
        pts = torch.from_numpy(make_clouds("ball", b, N, seed=b)).cuda()
        labels = torch.arange(b, device="cuda") % M.NUM_CLASSES

        def fused_step():
            logits, _ = M.get_model_training(pts, *gmm, None, params=p)
            M.get_loss(logits, labels).backward()
            p._flat.flat.grad = None

        def composed_step():
            F.cross_entropy(comp.logits(pts, gmm), labels).backward()
            for v in comp.v.values():
                for t in v[:4]:
                    t.grad = None
            pc._flat.flat.grad = None

        fused_step(), composed_step()
        peaks = (peak(fused_step), peak(composed_step))
        tf, tc = alternate(fused_step, composed_step, a.windows, a.reps)
        print(f"\n## B={b} N={N}: whole step (forward, cross-entropy, backward)")
        print(f"fused {tf:.2f} ms = {b / tf * 1e3:.0f} clouds/s   composition {tc:.2f} ms = {b / tc * 1e3:.0f} clouds/s   "
              f"allocation peak fused {peaks[0] / 2**20:.0f} MiB, composition {peaks[1] / 2**20:.0f} MiB")
        tr = next(v for k, v in p._trainers.items() if k[0] == "mfv_net")
        rows = []
        print(f"{'layer':20s} {'k':>2s} {'c':>4s} {'cout':>4s} {'r':>2s} {'fused ms':>9s} {'torch ms':>9s} {'ratio':>6s} "
              f"{'dW MACs/in-grid':>16s} {'dx MACs/in-grid':>16s}")
        for scope, fused, composed, (k, c, cout, r) in layer_cases(tr, comp, b):
            lf, lc = alternate(fused, composed, a.windows, a.reps)
            iw, idd, ig = ops.conv3d_bwd_macs(b, r, k, c, cout)
            rows.append(dict(layer=scope, k=k, c=c, cout=cout, r=r, fused_ms=lf, torch_ms=lc, weight_macs_ratio=iw / ig, data_macs_ratio=idd / ig))
            print(f"{scope:20s} {k:2d} {c:4d} {cout:4d} {r:2d} {lf:9.3f} {lc:9.3f} {lc / lf:6.2f} {iw / ig:16.2f} {idd / ig:16.2f}")
        result["batches"][b] = dict(step_ms=tf, step_clouds_s=b / tf * 1e3, torch_step_ms=tc, torch_clouds_s=b / tc * 1e3,
                                    peak_bytes=peaks[0], torch_peak_bytes=peaks[1], layers=rows)
        del tr, comp, p, pc
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
