"""SpiderCNN training at N=1024, B=16 and B=32: the spiderConv backward of csrc/spider.cu (spidercnn_cls_xyz.get_model_training)
against a torch autograd composition that materialises each layer's (B,N,k,C*T) conv input as the reference does (TF32 off).

  per layer   fanConv1..4: forward + backward time of one layer (spiderConv, group norm, ReLU, top-2 pooling, and the gradients of its
              variables and of its input activation; CUDA events, median of repeats after warm-up, the two paths alternated) and the
              rise of torch.cuda.max_memory_allocated over one forward + backward
  whole step  get_model_training + cross-entropy + backward, clouds/s; the composition runs the same head (training.mlp_training)
              behind the four composed layers

Prints the card name and power limit, then one JSON line.  Usage: python tools/spidercnn_train_timing.py [--reps 10] [--steps 10]"""
import argparse
import gc
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from scanobjectnn_b200 import ops
from scanobjectnn_b200 import spidercnn_cls_xyz as M
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import GN_EPS, TAYLOR_TERMS
from scanobjectnn_b200.training import mlp_training

N, K, T = 1024, M.NSAMPLE, M.TAYLOR_CHANNEL
LAYERS = [(3, 32), (32, 64), (64, 128), (128, 256)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def event_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def compose_layer(h, idx, delta, taylor, W, bias, gamma, beta):
    """one spiderConv + group norm + ReLU + top-2 as torch ops, with the (B,N,k,C*T) conv input materialised -> (h_out, pooled)"""
    b, n, c = h.shape
    cout = W.shape[-1]
    grouped = h[torch.arange(b, device=h.device)[:, None, None], idx.long()]                            # (B,N,k,C)
    X, Y, Z = (delta[..., i] for i in range(3))
    one = torch.ones_like(X)
    mono = torch.stack([X, Y, Z, X * Y * Z, X * Y, Y * Z, X * Z, one, X * X, Y * Y, Z * Z, X * X * Y, X * Y * Y, X * X * Z, X * Z * Z,
                        Y * Y * Z, Y * Z * Z, X * X * X, Y * Y * Y, Z * Z * Z], dim=-1)
    g = mono @ taylor                                                                                   # (B,N,k,T)
    conv_in = (grouped[..., None] * g[:, :, :, None, :]).reshape(b, n, K * c * T)
    y = conv_in @ W.reshape(K * c * T, cout) + bias
    G = min(16, cout)
    yt = y.reshape(b, n, G, cout // G)
    mean = yt.mean(dim=(1, 3), keepdim=True)
    var = ((yt - mean) ** 2).mean(dim=(1, 3), keepdim=True)
    z = torch.relu(((yt - mean) / torch.sqrt(var + GN_EPS)).reshape(b, n, cout) * gamma + beta)
    return z, torch.topk(z.permute(0, 2, 1), 2, dim=-1).values


def layer_params(p, l):
    sc = f"fanConv{l}/taylor"
    taylor = torch.cat([p[f"{sc}/{m}"].reshape(1, -1) for m in TAYLOR_TERMS]).clone().requires_grad_(True)
    return [taylor] + [p[f"{sc}/{v}"].clone().requires_grad_(True) for v in ("conv/weights", "conv/biases", "conv/gn/gamma", "conv/gn/beta")]


def fused_layer(b, l, x, dpool):
    """forward + backward of fanConv{l} on the libpsa ops (allocating, as a caller outside a trainer would)"""
    feat, fs, fu, idx, delta, taylor, W, bias, gamma, beta = x
    c, cout = LAYERS[l - 1]
    y = ops.spider_conv(delta, idx, feat, taylor, W, bias, fs, fu)
    scale, shift = ops.group_norm_affine(y, gamma, beta, min(16, cout), GN_EPS)
    pooled = ops.topk_pool(y, 2, scale, shift, relu=True)
    dy, dgamma, dbeta = ops.spider_gn_bwd(y, scale, shift, gamma, min(16, cout), dpool)
    db = dy.sum(dim=(0, 1))
    g = ops.spider_taylor_filter(delta, taylor)
    dW = ops.spider_conv_bwd_weight(idx, feat, g, dy, fs, fu)
    D, dg = ops.spider_conv_bwd_data(idx, feat, g, W, dy, fs, fu, want_D=l > 1)
    dtaylor = ops.spider_taylor_grad(delta, dg)
    if D is not None:
        pts = torch.zeros_like(feat, requires_grad=True)
        ops.group_point(pts, idx).backward(D)
    return pooled, dW, db, dtaylor, dgamma, dbeta


def per_layer(b, reps):
    res = {}
    p = M.init_params(seed=1, randomize_bn=True)
    xyz = torch.from_numpy(make_clouds("ball", b, N, seed=3)).cuda()
    with torch.no_grad():
        _, ep = M.get_model(xyz, False, params=p, return_end_points=True)
    idx = ep["idx"]
    delta = (ops.group_point(xyz, idx) - xyz.unsqueeze(2)).contiguous()
    rng = np.random.default_rng(0)
    for l, (c, cout) in enumerate(LAYERS, start=1):
        feat = xyz if l == 1 else ep[f"y{l - 1}"]
        fs, fu = (None, None) if l == 1 else (ep[f"scale{l - 1}"], ep[f"shift{l - 1}"])
        h = xyz if l == 1 else torch.relu(feat * fs[:, None] + fu[:, None])
        dpool = torch.tensor(rng.standard_normal((b, cout, 2)).astype(np.float32), device="cuda")
        taylor, W, bias, gamma, beta = p.spider(f"fanConv{l}/taylor")
        x = (feat, fs, fu, idx, delta, taylor, W, bias, gamma, beta)
        hc = h.detach().clone().requires_grad_(l > 1)
        prm = layer_params(p, l)

        def comp():
            _, pooled = compose_layer(hc, idx, delta, *prm)
            return torch.autograd.grad(pooled, prm + ([hc] if l > 1 else []), dpool)

        paths = {"composition": comp, "fused": lambda: fused_layer(b, l, x, dpool)}
        mem = {}
        for name, fn in paths.items():
            for _ in range(2):
                fn()
            gc.collect()
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            fn()
            torch.cuda.synchronize()
            mem[name] = (torch.cuda.max_memory_allocated() - base) / 2**20
        t = {name: [] for name in paths}
        for _ in range(reps):
            for name, fn in paths.items():
                t[name].append(event_ms(fn))
        res[f"fanConv{l}"] = {**{name: {"fwd_bwd_ms": float(np.median(t[name])), "peak_alloc_rise_mib": mem[name]} for name in paths},
                              "speedup": float(np.median(t["composition"]) / np.median(t["fused"]))}
        torch.cuda.empty_cache()
    return res


def composed_model(xyz, p, params_per_layer):
    b = xyz.shape[0]
    _, idx = ops.knn_point(K, xyz, xyz)
    delta = ops.group_point(xyz, idx) - xyz.unsqueeze(2)
    h, pools = xyz, []
    for prm in params_per_layer:
        h, pooled = compose_layer(h, idx, delta, *prm)
        pools.append(pooled)
    net = torch.cat(pools, dim=1).reshape(b, -1)
    net = torch.nn.functional.dropout(mlp_training(net, [("fc1", True)], None, p), 0.7, training=True)
    net = torch.nn.functional.dropout(mlp_training(net, [("fc2", True)], None, p), 0.7, training=True)
    return mlp_training(net, [("fc3", False)], None, p)


def whole_step(b, steps):
    xyz = torch.from_numpy(make_clouds("ball", b, N, seed=5)).cuda()
    labels = torch.randint(0, M.NUM_CLASSES, (b,), device="cuda")
    pf, pc = M.init_params(seed=2), M.init_params(seed=2)
    prm = [layer_params(pc, l) for l in range(1, 5)]

    def fused():
        if getattr(pf, "_flat", None) is not None:
            pf._flat.flat.grad = None
        M.get_loss(M.get_model_training(xyz, None, params=pf), labels).backward()

    def comp():
        M.get_loss(composed_model(xyz, pc, prm), labels).backward()

    out = {}
    for name, fn in (("fused", fused), ("composition", comp)):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ms = float(np.median([event_ms(fn) for _ in range(steps)]))
        out[name] = {"step_ms": ms, "clouds_per_s": b / ms * 1e3}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    c = card()
    print(f"card: {c}")
    res = {"card": c, "n": N}
    for b in (16, 32):
        res[f"B{b}"] = {"per_layer": per_layer(b, args.reps), "step": whole_step(b, args.steps)}
        print(f"B={b}: {json.dumps(res[f'B{b}'])}", file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
