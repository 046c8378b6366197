"""pointcnn_cls training at N=1024, B=32 (PointCNN/train.py's setting) and B=16: the fused training step (csrc/pointcnn_train.cu's stages
and backward, get_model_training) against a torch autograd composition that materialises the (B,P,N) distance matrix and every
(B,P,K,.) tensor (fp32, TF32 off, F.batch_norm(training=True, momentum=0.01), grouped F.conv2d for the depthwise layers).

Each side is captured as a CUDA graph and timed in alternating windows (CUDA events around `--reps` replays, median of `--windows`):
the whole step (forward, tiled cross-entropy, backward) in clouds/s, each X-Conv layer's forward + backward, the allocation peak of
each side's step, and psa_bn_finalize_rows on the B*P*K-row lifting layers, which launch ceil(C/32) blocks.  Prints the card and its
power limit, then one JSON line."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scanobjectnn_b200 import _lib  # noqa: E402
from scanobjectnn_b200 import pointcnn_cls as M  # noqa: E402
from scanobjectnn_b200.synthetic import make_clouds  # noqa: E402
from scanobjectnn_b200.tf_util import BN_EPS  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


# ---- the torch composition ----
def knn(pts, qrs, k, d):
    dist = (qrs[:, :, None, :] - pts[:, None, :, :]).square().sum(-1)                 # (B, P, N)
    return torch.topk(-dist, k * d, dim=-1).indices[:, :, ::d]


class Composition(torch.nn.Module):
    """pointcnn_cls in training mode from torch ops on a copy of the store's variables"""

    def __init__(self, params):
        super().__init__()
        self.v = torch.nn.ParameterDict({k.replace("/", "|"): torch.nn.Parameter(v.detach().clone())
                                         for k, v in params.items() if not k.endswith(("moving_mean", "moving_variance"))})
        self.mov = {k: v.detach().clone() for k, v in params.items() if k.endswith(("moving_mean", "moving_variance"))}

    def p(self, name):
        return self.v[name.replace("/", "|")]

    def bn(self, x, layer):
        c = x.shape[-1]
        y = F.batch_norm(x.reshape(-1, c), self.mov[f"{layer}_bn/moving_mean"], self.mov[f"{layer}_bn/moving_variance"], self.p(f"{layer}_bn/gamma"),
                         self.p(f"{layer}_bn/beta"), training=True, momentum=0.01, eps=BN_EPS)
        return y.reshape(x.shape)

    def dense(self, x, layer, var="kernel"):
        w = self.p(f"{layer}/{var}")
        return self.bn(F.elu(x @ w.reshape(-1, w.shape[-1])), layer)

    def xconv(self, l, pts, fts):
        tag, k, d, p, c, c_pts, c_prev, dm, glob = M.layer_table()[l]
        p = pts.shape[1] if p == -1 else p
        qrs = pts[:, :p]
        B = pts.shape[0]
        idx = knn(pts, qrs, k, d)
        bi = torch.arange(B, device=pts.device)[:, None, None]
        local = pts[bi, idx] - qrs[:, :, None, :]
        lifted = self.dense(self.dense(local, f"{tag}nn_fts_from_pts_0"), f"{tag}nn_fts_from_pts")
        Fm = lifted if fts is None else torch.cat([lifted, fts[bi, idx]], dim=-1)
        X = self.bn(F.elu(local.reshape(B, p, -1) @ self.p(f"{tag}X_0/kernel").reshape(3 * k, k * k)), f"{tag}X_0")
        for name, act in (("X_1", True), ("X_2", False)):
            w = self.p(f"{tag}{name}/depthwise_weights")
            y = F.conv2d(X.reshape(B, p, k, k).permute(0, 3, 1, 2), w.permute(2, 3, 0, 1).reshape(k * k, 1, 1, k), groups=k)
            y = y[..., 0].permute(0, 2, 1)
            X = self.bn(F.elu(y) if act else y, f"{tag}{name}")
        fts_X = X.reshape(B, p, k, k) @ Fm
        wdw = self.p(f"{tag}fts_conv/depthwise_kernel")
        cin = wdw.shape[2]
        dw = F.conv2d(fts_X.permute(0, 3, 1, 2), wdw.permute(2, 3, 0, 1).reshape(cin * dm, 1, 1, k), groups=cin)[..., 0].permute(0, 2, 1)
        out = self.dense(dw, f"{tag}fts_conv", "pointwise_kernel")
        if glob:
            out = torch.cat([self.dense(self.dense(qrs, f"{tag}fts_global_0"), f"{tag}fts_global"), out], dim=-1)
        return qrs, out

    def forward(self, pts, mask):
        fts = None
        for l in range(4):
            pts, fts = self.xconv(l, pts, fts)
        net = self.dense(self.dense(fts, "fc0"), "fc1") * mask.view(fts.shape[0], fts.shape[1], -1)
        return net @ self.p("logits/kernel") + self.p("logits/bias")


# ---- timing ----
def graph_of(fn, warm=3):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(warm):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def alternate(graphs, reps, windows):
    """median ms per replay of each graph, windows alternating between them"""
    times = [[] for _ in graphs]
    for _ in range(windows):
        for i, g in enumerate(graphs):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                g.replay()
            b.record()
            b.synchronize()
            times[i].append(a.elapsed_time(b) / reps)
    return [sorted(t)[len(t) // 2] for t in times]


def peak_of(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def run(b, n, reps, windows):
    torch.manual_seed(0)
    p = M.init_params(seed=1, randomize_bn=True)
    x = torch.from_numpy(make_clouds("ball", b, n, seed=2)).cuda()
    label = torch.arange(b, device="cuda") % M.NUM_CLASSES
    comp = Composition(p).cuda()
    res = {"B": b, "N": n}

    def fused_step():
        if getattr(p, "_flat", None) is not None:
            p._flat.flat.grad = None
        M.get_loss(M.get_model_training(x, params=p), label).backward()

    mask = torch.empty((b * 128, M.FC[-1]), device="cuda")

    def comp_step():
        comp.zero_grad(set_to_none=True)
        mask.bernoulli_(M.DROPOUT_KEEP).mul_(1.0 / M.DROPOUT_KEEP)
        M.get_loss(comp(x, mask), label).backward()

    res["peak_fused_MiB"] = peak_of(fused_step)            # the trainer's buffers included (first call)
    res["peak_torch_MiB"] = peak_of(comp_step)
    gf, gc = graph_of(fused_step), graph_of(comp_step)
    tf, tc = alternate([gf, gc], reps, windows)
    res.update(step_ms_fused=tf, step_ms_torch=tc, clouds_per_s_fused=b / tf * 1e3, clouds_per_s_torch=b / tc * 1e3)

    # per layer: forward + backward of one X-Conv layer on the run's inputs, a fixed upstream gradient
    tr = p._trainers[("pointcnn_cls", b, n)]
    layers = []
    pts_c, fts_c = x, None
    for i, L in enumerate(tr.layers):
        pts = x if i == 0 else tr.layers[i - 1]["qrs"]
        fts = None if i == 0 else tr.layers[i - 1]["out"]
        dout = torch.randn(L["out"].shape, device="cuda")
        d_fts = None if fts is None else torch.empty_like(fts)
        fin = pts_c.detach()
        fc = None if fts_c is None else fts_c.detach().requires_grad_(True)

        def fused_layer(L=L, pts=pts, fts=fts, dout=dout, d_fts=d_fts):
            tr.layer_forward(L, pts, fts)
            tr.layer_backward(L, dout, d_fts)

        def comp_layer(i=i, fin=fin, fc=fc, dout=dout):
            comp.zero_grad(set_to_none=True)
            _, out = comp.xconv(i, fin, fc)
            out.backward(dout.view(out.shape))

        gl, gcl = graph_of(fused_layer), graph_of(comp_layer)
        lf, lc = alternate([gl, gcl], reps, windows)
        with torch.no_grad():
            pts_c, fts_c = comp.xconv(i, pts_c, fts_c)
        # psa_bn_finalize_rows on the B*P*K-row lifting layers (ceil(C/32) blocks)
        lib, bn = _lib.load(), L["bn"]["pts1"]

        def fin_rows(bn=bn):
            _lib.check(lib.psa_bn_finalize_rows(bn["rows"], bn["C"], _lib.ptr(bn["a"]), _lib.ptr(bn["gamma"]), _lib.ptr(bn["beta"]), C.c_float(1.0),
                                                None, None, _lib.ptr(bn["s"]), _lib.ptr(bn["t"]), _lib.ptr(bn["mean_inv"]), _lib.stream()),
                       "bn_finalize_rows")

        (tfin,) = alternate([graph_of(fin_rows)], reps, windows)
        layers.append({"layer": L["tag"].rstrip("_"), "fwd_bwd_ms_fused": lf, "fwd_bwd_ms_torch": lc, "bn_finalize_rows_ms_per_call": tfin,
                       "bn_finalize_rows_calls": 2, "rows": bn["rows"], "C": bn["C"]})
    res["layers"] = layers
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[32, 16])
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--windows", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pointcnn_train_timing: needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    print("card:", card())
    out = []
    for b in a.batches:
        r = run(b, a.n, a.reps, a.windows)
        print(f"B={b} N={a.n}: fused {r['clouds_per_s_fused']:.0f} clouds/s ({r['step_ms_fused']:.2f} ms), torch {r['clouds_per_s_torch']:.0f} "
              f"clouds/s ({r['step_ms_torch']:.2f} ms); peak {r['peak_fused_MiB']:.0f} vs {r['peak_torch_MiB']:.0f} MiB")
        for L in r["layers"]:
            print(f"  {L['layer']}: fwd+bwd fused {L['fwd_bwd_ms_fused']:.3f} ms, torch {L['fwd_bwd_ms_torch']:.3f} ms; "
                  f"bn_finalize_rows ({L['rows']} x {L['C']}) {L['bn_finalize_rows_ms_per_call']:.3f} ms x {L['bn_finalize_rows_calls']}")
        out.append(r)
    print(json.dumps({"card": card(), "results": out}))


if __name__ == "__main__":
    main()
