"""Tensor-core kNN graph (psa_knn_graph_ws, csrc/knn_tc.cu) at B=32, N=2048, k=20 on four cloud types: time per call with CUDA
events, number of rows that went to the exhaustive kernel, and the fp32 kernel (psa_knn_graph) beside it: time, index equality."""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from scanobjectnn_b200 import _lib
from scanobjectnn_b200.synthetic import make_clouds


def median_us(run, warmup, reps):
    for _ in range(warmup):
        assert run() == 0
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); run(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    return sorted(ts)[reps // 2]


lib = _lib.load()
B, N, K = 32, 2048, 20
out = {}
for name, x in (("c64_gauss", torch.randn((B, N, 64), device="cuda")), ("c3_ball", torch.from_numpy(make_clouds("ball", B, N, seed=5)).cuda()),
                ("c64_relu", torch.relu(torch.randn((B, N, 64), device="cuda"))),
                # a feature cloud far from the origin (|x|^2 ~ 50 x the neighbour distances), like DGCNN's post-ReLU EdgeConv outputs
                ("c64_offset", torch.relu(torch.randn((B, N, 64), device="cuda") * 0.3 + 2.0))):
    c = x.shape[2]
    need = lib.psa_knn_graph_workspace_bytes(B, N, c, K)
    ws = torch.zeros(need // 4 + 1, dtype=torch.float32, device="cuda")
    idx = torch.empty((B, N, K), dtype=torch.int32, device="cuda")
    ref = torch.empty_like(idx)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    vp = lambda t: C.c_void_p(t.data_ptr())
    tc_us = median_us(lambda: lib.psa_knn_graph_ws(B, N, c, K, vp(x), vp(idx), vp(ws), C.c_size_t(need), st), 3, 7)
    npad = (N + 127) // 128 * 128
    off = (B * (npad // 128) * 49152 + ((B * npad * 4 + 255) & ~255) + ((B * N * 4 + 255) & ~255)) // 4
    flagged = int(ws[off:off + 1].view(torch.int32).item())
    fp32_us = median_us(lambda: lib.psa_knn_graph(B, N, c, K, vp(x), vp(ref), st), 2, 5)
    out[name] = {"tc_us": tc_us, "fp32_us": fp32_us, "rows_to_exhaustive_kernel": flagged, "rows": B * N,
                 "equal": bool(torch.equal(idx, ref))}
print(json.dumps(out))
