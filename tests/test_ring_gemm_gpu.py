"""The shared ring GEMM (csrc/ring_gemm.cuh) and its FMA fallback through its ops -- conv3d, PointCNN's dense layer, spiderConv and
the dense layer of psa_shared_mlp -- called through the C ABI so that the test owns every buffer, against float64 at the plan's edges:

* every call is poisoned around: inputs are slices of NaN-filled buffers (NaN columns on both sides, NaN rows past the end), the
  output is a slice of a NaN-filled wider buffer, the workspace is NaN-filled and has NaN bytes past what it asked for.  Only the
  owned output may change, and it must meet the contract;
* before a dense or spiderConv launch on the tensor cores, the same kernel runs once over +inf operands on every SM, so that the
  shared memory the launch does not stage (rows past the last tile's end, columns past K) holds inf and NaN and must be masked;
* conv3d units with no K blocks, ragged and padded tiles at shapes only the C ABI reaches, with more units than SMs on both tile
  widths, the fp16x2 range guard at its edges, and row independence of the dense layer.

conv3d runs without its ReLU, which would turn a NaN into 0.  The shapes are named by the plans restated in tests/restate.py."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import mfv_oracle as mo
from oracle import pointcnn_oracle as po
from oracle import spidercnn_oracle as so
from scanobjectnn_b200 import _lib, ops
from scanobjectnn_b200.tf_util import VariableStore

from . import gpu_util as G
from . import restate as R

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
NAN_BITS = 0x7FC00000                                                         # torch.full's NaN
P = _lib.ptr


@contextlib.contextmanager
def _mode(m):
    ops.set_mlp_mode(m)
    try:
        yield
    finally:
        ops.set_mlp_mode(0)


def _inside(t):
    """a copy of t inside a NaN-filled buffer, 256 bytes after its start and 256 bytes before its end"""
    buf = torch.full((t.numel() + 128,), NAN, device="cuda")
    buf[64:64 + t.numel()] = t.reshape(-1)
    return buf[64:64 + t.numel()].view(t.shape)


def _columns_of(t):
    """t (rows, cols) as the column slice [32, 32 + cols) of a NaN-filled (rows + 3, cols + 64) buffer -> (view, buffer)"""
    rows, cols = t.shape
    buf = torch.full((rows + 3, cols + 64), NAN, device="cuda")
    buf[:rows, 32:32 + cols] = t
    return buf[:rows, 32:32 + cols], buf


def _owned(view, buf, what):
    """the values the call wrote in `view`; every other element of `buf` must still be the NaN it was filled with"""
    got = view.clone()
    view.fill_(NAN)
    bad = int((buf.view(torch.int32) != NAN_BITS).sum())
    assert bad == 0, f"{what}: {bad} elements written outside the output"
    return got


class _Ws:
    """a NaN-filled workspace of the bytes the current mode asks for, and 4 KB more that must stay NaN; word `flag_word` is the range
    flag"""

    def __init__(self, need, flag_word=0):
        self.need, self.flag_word = int(need), flag_word
        self.buf = torch.full((self.need // 4 + 1024,), NAN, device="cuda")

    def args(self):
        return P(self.buf), C.c_size_t(self.need)

    def flag(self):
        return int(self.buf[self.flag_word:self.flag_word + 1].view(torch.int32))

    def check_tail(self, what):
        assert bool((self.buf[self.need // 4:].view(torch.int32) == NAN_BITS).all()), f"{what}: wrote past its workspace"


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---------------------------------------------------------------------------------------------------------------------
# the three ops, each as case (inputs and float64 reference) -> call
# ---------------------------------------------------------------------------------------------------------------------
class Conv:
    """psa_conv3d_infer on voxel-major rows (B r^3, c), batch norm folded, no ReLU"""
    name = "conv3d"

    def __init__(self, b, r, k, c, n, seed):
        self.b, self.r, self.k, self.c, self.n, self.rows = b, r, k, c, n, b * r ** 3
        self.p = VariableStore(device="cuda", seed=seed)
        self.p.add_conv3d("c", k, c, n, randomize_bn=True)
        gen = torch.Generator(device="cuda").manual_seed(seed)
        self.x = torch.randn((self.rows, c), generator=gen, device="cuda")
        W, sc, sh, _ = self.p.folded("c")
        self.W, self.scale, self.shift = W.clone(), sc, sh

    def want(self, x=None):
        b, r = self.b, self.r
        grid = (self.x if x is None else x).double().reshape(r ** 3, b, -1).permute(1, 2, 0).reshape(b, -1, r, r, r)
        y = mo.conv3d(grid, self.p, "c", relu=False)
        return y.reshape(b, self.n, r ** 3).permute(2, 0, 1).reshape(self.rows, self.n)

    def need(self):
        return _lib.load().psa_conv3d_workspace_bytes(self.b, self.r, self.k, self.c, self.n)

    def call(self, ws, x=None, W=None):
        x, _ = _columns_of(self.x if x is None else x)
        out, obuf = _columns_of(torch.full((self.rows, self.n), NAN, device="cuda"))
        Wi, sc, sh = _inside(self.W if W is None else W), _inside(self.scale), _inside(self.shift)
        rc = _lib.load().psa_conv3d_infer(self.b, self.r, self.k, self.c, self.n, P(x), x.stride(0), P(Wi), P(sc), P(sh), 0, P(out),
                                          out.stride(0), *ws.args(), _lib.stream())
        assert rc == 0, _lib.load().psa_last_error()
        return _owned(out, obuf, self.label())

    def label(self):
        return f"conv3d b={self.b} r={self.r} k={self.k} {self.c}->{self.n}"

    def plan(self):
        return R.conv_plan(self.b, self.r, self.k, self.c, self.n, 2)


class Dense:
    """psa_dense_elu_affine: elu(x . W + bias) * scale + shift"""
    name = "dense"

    def __init__(self, rows, K, N, seed):
        self.rows, self.K, self.n = rows, K, N
        g = torch.Generator().manual_seed(seed)
        self.x = torch.randn((rows, K), generator=g).cuda()
        self.W = (torch.randn((K, N), generator=g) / np.sqrt(K)).cuda()
        self.scale = (torch.rand(N, generator=g) * 2 + 0.5).cuda()
        self.shift = (torch.randn(N, generator=g) * 0.1).cuda()
        self.bias = (torch.randn(N, generator=g) * 0.1).cuda()

    def want(self, x=None):
        x = self.x if x is None else x
        y = G.npy(x).astype(np.float64) @ G.npy(self.W).astype(np.float64) + G.npy(self.bias)
        return torch.from_numpy(po.elu(y) * G.npy(self.scale) + G.npy(self.shift))

    def need(self):
        return _lib.load().psa_dense_elu_affine_workspace_bytes(self.rows, self.K, self.n)

    def call(self, ws, x=None, W=None):
        x, _ = _columns_of(self.x if x is None else x)
        out, obuf = _columns_of(torch.full((x.shape[0], self.n), NAN, device="cuda"))
        Wi, bi, sc, sh = _inside(self.W if W is None else W), _inside(self.bias), _inside(self.scale), _inside(self.shift)
        rc = _lib.load().psa_dense_elu_affine(x.shape[0], self.K, self.n, P(x), x.stride(0), P(Wi), P(bi), P(sc), P(sh), P(out),
                                              out.stride(0), *ws.args(), _lib.stream())
        assert rc == 0, _lib.load().psa_last_error()
        return _owned(out, obuf, self.label())

    def label(self):
        return f"dense {self.rows}x{self.K}x{self.n}"

    def plan(self):
        return R.pd_plan(self.rows, self.K, self.n, 2)


class Spider:
    """psa_spider_conv_infer with the previous layer's group-norm affine, on random in-cloud neighbours"""
    name = "spider"

    def __init__(self, b, npts, c, k, t, n, seed):
        self.b, self.npts, self.c, self.k, self.t, self.n, self.rows = b, npts, c, k, t, n, b * npts
        gen = torch.Generator(device="cuda").manual_seed(seed)
        xyz = torch.rand((b, npts, 3), generator=gen, device="cuda") * 2 - 1
        self.idx = torch.randint(0, npts, (b, npts, k), generator=gen, device="cuda", dtype=torch.int32)
        self.delta = (so.group_point(xyz, self.idx) - xyz[:, :, None, :]).contiguous()
        self.feat = torch.randn((b, npts, c), generator=gen, device="cuda")
        self.fs = torch.rand((b, c), generator=gen, device="cuda") * 2 - 0.5
        self.fu = torch.rand((b, c), generator=gen, device="cuda") - 0.5
        self.p = VariableStore(device="cuda", seed=seed)
        self.p.add_spider_conv("spider", c, n, k, t)
        self.p["spider/biases"] = torch.rand((1, 1, 1, t), generator=gen, device="cuda") - 0.5
        self.p["spider/conv/biases"] = torch.rand(n, generator=gen, device="cuda") - 0.5
        self.taylor, W, self.bias, _, _ = self.p.spider("spider")
        self.W = W.clone()

    def want(self, delta=None):
        """float64 pre-norm y (rows, n), one cloud at a time"""
        delta = self.delta if delta is None else delta
        out = []
        for i in range(self.b):
            h = torch.relu(self.feat[i:i + 1].double() * self.fs[i:i + 1].double()[:, None] + self.fu[i:i + 1].double()[:, None])
            out.append(so.spider_conv_prenorm(h, self.idx[i:i + 1], delta[i:i + 1].double(), self.p, "spider"))
        return torch.cat(out).reshape(self.rows, self.n)

    def need(self):
        return _lib.load().psa_spider_conv_workspace_bytes(self.b, self.npts, self.c, self.k, self.t, self.n)

    def call(self, ws, delta=None, W=None):
        d, f, fs, fu = _inside(self.delta if delta is None else delta), _inside(self.feat), _inside(self.fs), _inside(self.fu)
        tay, Wi, bi = _inside(self.taylor), _inside(self.W if W is None else W), _inside(self.bias)
        ybuf = torch.full((self.rows * self.n + 128,), NAN, device="cuda")
        y = ybuf[64:64 + self.rows * self.n]
        rc = _lib.load().psa_spider_conv_infer(self.b, self.npts, self.c, self.k, self.t, self.n, P(d), P(self.idx), P(f), P(fs), P(fu),
                                               P(tay), P(Wi), P(bi), P(y), *ws.args(), _lib.stream())
        assert rc == 0, _lib.load().psa_last_error()
        return _owned(y, ybuf, self.label()).view(self.rows, self.n)

    def label(self):
        return f"spider b={self.b} n={self.npts} c={self.c} k={self.k} T={self.t} ->{self.n}"

    def plan(self):
        return R.spider_plan(self.b, self.npts, self.c, self.k, self.t, self.n)


class Mlp:
    """a one-layer psa_shared_mlp (psa_shared_mlp_grouped with group_rows): (x . W [+ group_add[r / group_rows]]) * scale + shift,
    no ReLU, then the max over runs of pool_k rows; x starts `offset` floats past a 16-byte boundary"""
    name = "mlp"

    def __init__(self, rows, K, N, pool_k, offset=0, group_rows=0, seed=0):
        self.rows, self.K, self.n, self.pool_k, self.offset, self.group_rows = rows, K, N, pool_k, offset, group_rows
        g = torch.Generator().manual_seed(seed)
        self.x = torch.randn((rows, K), generator=g).cuda()
        self.W = (torch.randn((K, N), generator=g) / np.sqrt(K)).cuda()
        self.scale = (torch.rand(N, generator=g) * 2 + 0.5).cuda()
        self.shift = (torch.randn(N, generator=g) * 0.1).cuda()
        self.gadd = torch.randn((rows // group_rows, N), generator=g).cuda() if group_rows else None

    def want(self, x=None):
        y = G.npy(self.x if x is None else x).astype(np.float64) @ G.npy(self.W).astype(np.float64)
        if self.gadd is not None:
            y += np.repeat(G.npy(self.gadd).astype(np.float64), self.group_rows, axis=0)
        y = y * G.npy(self.scale) + G.npy(self.shift)
        return torch.from_numpy(y.reshape(self.rows // self.pool_k, self.pool_k, self.n).max(1))

    def mlp(self, W=None):
        return ops.MlpParams([(_inside(self.W if W is None else W), _inside(self.scale), _inside(self.shift), False)])

    def need(self):
        return _lib.load().psa_shared_mlp_workspace_bytes(self.rows, self.mlp().ref)

    def flag_word(self):
        return (self.need() - 256) // 4                                       # the word region sits at the workspace's end

    def call(self, ws, x=None, W=None):
        x = self.x if x is None else x
        xbuf = torch.full((x.numel() + 128,), NAN, device="cuda")
        xi = xbuf[64 + self.offset:64 + self.offset + x.numel()].view(x.shape)
        xi.copy_(x)
        obuf = torch.full(((self.rows // self.pool_k) * self.n + 128,), NAN, device="cuda")
        out = obuf[64:64 + (self.rows // self.pool_k) * self.n]
        mlp, lib = self.mlp(W), _lib.load()
        if self.gadd is None:
            rc = lib.psa_shared_mlp(self.rows, self.pool_k, P(xi), mlp.ref, P(out), *ws.args(), _lib.stream())
        else:
            rc = lib.psa_shared_mlp_grouped(self.rows, self.group_rows, P(xi), mlp.ref, P(_inside(self.gadd)), P(out), *ws.args(),
                                            _lib.stream())
        assert rc == 0, lib.psa_last_error()
        return _owned(out, obuf, self.label()).view(self.rows // self.pool_k, self.n)

    def label(self):
        ga = f" group_rows={self.group_rows}" if self.group_rows else ""
        return f"shared_mlp {self.rows}x{self.K}x{self.n} pool {self.pool_k} offset {self.offset}{ga}"

    def plan(self):
        tiles = (self.rows + 127) // 128
        Nt = 128 if R.wide_tiles(tiles, self.n) else 64
        return dict(Nt=Nt, units=tiles * (self.n // Nt))


# ---------------------------------------------------------------------------------------------------------------------
# stale shared memory
# ---------------------------------------------------------------------------------------------------------------------
def _stale_inf(op, nc):
    """One launch of op's ring kernel, in the current mode and at tile width 64 nc, over +inf activations and weights on every SM
    (units >= 132) through four K blocks (every ring stage).  What it leaves in shared memory is inf, or NaN where the bf16x3 rerun
    split an inf weight; a later launch reads those bytes wherever it stages nothing."""
    rows, K, N = 2 * R.PLAN_SMS * 128, 256, 64 * nc
    ones = torch.ones(N, device="cuda")
    lib = _lib.load()
    if op.name == "dense":
        x, W = torch.full((rows, K), INF, device="cuda"), torch.full((K, N), INF, device="cuda")
        out = torch.empty((rows, N), device="cuda")
        ws = _Ws(lib.psa_dense_elu_affine_workspace_bytes(rows, K, N))
        rc = lib.psa_dense_elu_affine(rows, K, N, P(x), K, P(W), P(None), P(ones), P(ones), P(out), N, *ws.args(), _lib.stream())
    elif op.name == "mlp":
        x, W = torch.full((rows, K), INF, device="cuda"), torch.full((K, N), INF, device="cuda")
        out = torch.empty((rows, N), device="cuda")
        mlp = ops.MlpParams([(W, ones, ones, False)])
        ws = _Ws(lib.psa_shared_mlp_workspace_bytes(rows, mlp.ref))
        rc = lib.psa_shared_mlp(rows, 1, P(x), mlp.ref, P(out), *ws.args(), _lib.stream())
    else:                                                                     # spider: c = 64, k = 1, T = 4, g = 1
        c, t = 64, 4
        feat, W = torch.full((rows, c), INF, device="cuda"), torch.full((t * c, N), INF, device="cuda")
        taylor = torch.zeros((20, t), device="cuda")
        taylor[7] = 1.0                                                       # the constant term
        delta, idx = torch.zeros((rows, 3), device="cuda"), torch.zeros((rows,), device="cuda", dtype=torch.int32)
        y = torch.empty((rows, N), device="cuda")
        ws = _Ws(lib.psa_spider_conv_workspace_bytes(1, rows, c, 1, t, N))
        rc = lib.psa_spider_conv_infer(1, rows, c, 1, t, N, P(delta), P(idx), P(feat), P(None), P(None), P(taylor), P(W), P(ones), P(y),
                                       *ws.args(), _lib.stream())
    assert rc == 0, lib.psa_last_error()


def _run(op, mode, **inputs):
    """op's call in `mode` on a fresh poisoned workspace, after _stale_inf for the ring ops that mask stale bytes; in mode 0 a
    clean call must leave the range flag down (the fp16x2 result stands).  -> (output, workspace)"""
    with _mode(mode):
        ws = _Ws(op.need(), op.flag_word() if op.name == "mlp" else 0)
        if mode != 1 and op.name != "conv3d":                                # conv3d zero-fills every staged byte itself
            _stale_inf(op, op.plan()["Nt"] // 64)
        y = op.call(ws, **inputs)
        ws.check_tail(op.label())
    return y, ws


def _check(op, mode, want=None, **inputs):
    y, ws = _run(op, mode, **inputs)
    if mode == 0:
        assert ws.flag() == 0, f"{op.label()}: range flag {ws.flag():#x} after in-range operands (the fp16x2 result must stand)"
    want = op.want() if want is None else want
    err = G.contract_close(G.npy(y), G.npy(want), f"{op.label()} mode {mode}")
    print(f"[ring] {op.label()} mode {mode}: plan {_describe(op)}, max|err| = {err:.2e}")
    return y


def _describe(op):
    p = op.plan()
    return ", ".join(f"{k}={p[k]}" for k in ("Np", "Nt", "splits", "units") if k in p)


MODES = (0, 1, 2)


def _ids(cases):
    return [f"{k}-{'x'.join(map(str, s))}" for k, s in cases]


# ---------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", [64, 128])
def test_conv3d_units_without_k_blocks(c):
    """b = 128, r = 2, k = 3: 8 one-voxel tiles with 8 active taps.  c = 64 plans 13 splits, so 5 units of every tile have no K
    block and must still write a zero partial into the NaN-filled workspace; c = 128 plans 16 splits over 16 active blocks, one
    block per unit (tests/test_ring_gemm_plan_cpu.py: no c >= 128 plan has an empty unit)"""
    op = Conv(128, 2, 3, c, 64, seed=c)
    p = op.plan()
    nb = R.conv_unit_blocks(op.b, op.r, op.k, op.c, p["splits"])
    if c == 64:
        assert p["splits"] == 13 and all(row.count(0) == 5 for row in nb)
    else:
        assert p["splits"] == 16 and all(row == [1] * 16 for row in nb)
    want = op.want()
    for m in MODES:
        _check(op, m, want)


RAGGED = [
    # dense: rows % 128 in {1, 127}; K < 64, K % 64 != 0; N in {1, 63, 65, 129, 192}; more units than SMs on 64- and 128-wide tiles
    ("dense", (129, 4, 1)), ("dense", (255, 60, 63)), ("dense", (17025, 60, 65)), ("dense", (6017, 100, 129)), ("dense", (4223, 68, 192)),
    ("dense", (255, 132, 65)),
    # conv3d: c_out % 64 = 32 (Np padded), r in {1, 2}, a split plan, more units than SMs on 64- and 128-wide tiles
    ("conv", (255, 1, 3, 64, 32)), ("conv", (129, 1, 1, 64, 96)), ("conv", (100, 2, 3, 64, 32)), ("conv", (17025, 1, 3, 64, 96)),
    ("conv", (17023, 1, 5, 128, 32)),
    # spider: c = 32, one K block spanning two (j, t) slices; more units than SMs on 64- and 128-wide tiles
    ("spider", (1, 255, 32, 3, 2, 64)), ("spider", (1, 129, 32, 5, 2, 128)), ("spider", (3, 5675, 32, 4, 3, 64)),
    ("spider", (3, 5675, 32, 4, 3, 128)),
]
_OPS = {"dense": Dense, "conv": Conv, "spider": Spider}


def test_ragged_cases_cover_both_tile_widths_past_one_wave():
    """per op and tile width, at least one RAGGED case with more units than the 132 SMs the plans assume"""
    seen = set()
    for kind, shape in RAGGED:
        if kind == "conv":
            p = R.conv_plan(*shape, 2)
        elif kind == "dense":
            p = R.pd_plan(*shape, 2)
        else:
            p = R.spider_plan(*shape)
        if p["units"] > R.PLAN_SMS:
            seen.add((kind, p["Nt"]))
    assert seen == {(k, w) for k in _OPS for w in (64, 128)}


@pytest.mark.parametrize("kind,shape", RAGGED, ids=_ids(RAGGED))
def test_ragged_and_padded_tiles_match_float64(kind, shape):
    op = _OPS[kind](*shape, seed=sum(shape))
    want = op.want()
    for m in MODES:
        _check(op, m, want)


def _guarded(op, **inputs):
    """modes 0 and 2 on the same inputs: mode 0 must have raised its flag and returned mode 2's bits"""
    y0, ws = _run(op, 0, **inputs)
    assert ws.flag() != 0, f"{op.label()}: the range guard did not fire"
    y2, _ = _run(op, 2, **inputs)
    return y0, y2


def _overflowing(op, row):
    """op's inputs with row `row` beyond the fp16 range: x = 1e5, or for spiderConv a neighbour offset of 100 (|g| ~ 1e6)"""
    if op.name == "spider":
        big = op.delta.clone()
        big.view(op.rows, op.k, 3)[row] = 100.0
        return {"delta": big}
    big = op.x.clone()
    big[row] = 1e5
    return {"x": big}


OVERFLOW = [("conv", (17025, 1, 3, 64, 96)), ("dense", (17025, 60, 65)), ("dense", (6017, 100, 129)), ("spider", (3, 5675, 32, 4, 3, 128))]


@pytest.mark.parametrize("kind,shape", OVERFLOW, ids=_ids(OVERFLOW))
def test_overflow_in_one_row_of_the_last_tile(kind, shape):
    """the last row, alone in the last tile, beyond the fp16 range, in a launch whose CTAs walk several units: the fp16x2 pass raises
    the flag and the bf16x3 rerun rewrites every output, bit for bit mode 2, within the contract"""
    op = _OPS[kind](*shape, seed=sum(shape))
    assert op.plan()["units"] > R.PLAN_SMS and op.rows % 128 == 1
    big = _overflowing(op, -1)
    y0, y2 = _guarded(op, **big)
    assert _bits_equal(y0, y2)
    G.contract_close(G.npy(y0), G.npy(op.want(**big)), f"{op.label()} last row beyond fp16")


INF_WEIGHT = [("conv", (128, 2, 3, 64, 64)), ("dense", (255, 60, 65)), ("spider", (1, 255, 32, 3, 2, 64))]


@pytest.mark.parametrize("kind,shape", INF_WEIGHT, ids=_ids(INF_WEIGHT))
def test_non_finite_weight_reruns_on_bf16x3(kind, shape):
    """one inf weight: the image's non-finite-weight word sends mode 0 to the bf16x3 rerun, so mode 0 returns mode 2's bits (NaN
    included); its column is not finite, every other column meets the contract"""
    op = _OPS[kind](*shape, seed=sum(shape))
    W = op.W.clone()
    col = op.n // 2 + 1
    W.view(-1, op.n)[W.view(-1, op.n).shape[0] // 2, col] = INF             # conv3d: the centre tap
    want = op.want()
    y0, y2 = _guarded(op, W=W)
    assert _bits_equal(y0, y2)
    assert not bool(torch.isfinite(y0[:, col]).all())
    rest = [j for j in range(op.n) if j != col]
    G.contract_close(G.npy(y0[:, rest]), G.npy(want[:, rest]), f"{op.label()} inf weight, other columns")


@pytest.mark.parametrize("kind,shape", INF_WEIGHT, ids=_ids(INF_WEIGHT))
def test_a_clean_call_after_an_overflow_keeps_the_fp16x2_result(kind, shape):
    """clean, overflowing, clean on one workspace: the flag raised by the second call is cleared before the third, which returns
    the first call's bits.  Mode 2 differs from mode 0 on the clean input, so an inherited flag would show."""
    op = _OPS[kind](*shape, seed=sum(shape) + 1)
    with _mode(0):
        ws = _Ws(op.need())
        first = op.call(ws)
        assert ws.flag() == 0
        op.call(ws, **_overflowing(op, 0))
        assert ws.flag() != 0, f"{op.label()}: the range guard did not fire"
        third = op.call(ws)
        assert ws.flag() == 0
    y2, _ = _run(op, 2)
    assert not _bits_equal(first, y2), "mode 0 and mode 2 agree bit for bit: the check has no teeth"
    assert _bits_equal(third, first)


@pytest.mark.parametrize("mode", MODES)
def test_dense_rows_are_independent(mode):
    """the dense plan depends on N alone, and each output has a fixed summation order: the first R rows of a run over R + 300 rows
    are bit for bit a run over R rows, whose last tile holds 127 rows over stale shared memory"""
    R_ = 4223
    long = Dense(R_ + 300, 60, 65, seed=11)
    short = Dense(R_, 60, 65, seed=11)
    short.x, short.W, short.scale, short.shift, short.bias = long.x[:R_], long.W, long.scale, long.shift, long.bias
    assert short.plan()["Nt"] == long.plan()["Nt"] and R_ % 128 == 127
    want = long.want()
    a = _check(long, mode, want)
    b = _check(short, mode, want[:R_])
    assert _bits_equal(a[:R_], b)


MLP = [
    # rows % 128 in {1, 127}; K in {32, 99, 131} (99, 131: 4-byte staging); x off its 16-byte boundary; N in {64, 128, 256}
    (129, 32, 64, 1, 0), (255, 99, 128, 1, 0), (4223, 131, 256, 1, 0), (4223, 32, 128, 1, 1),
    # pool_k in {32, 64, 128, 256} (256: the ordered-int atomicMax between its fill and decode)
    (4096, 99, 128, 32, 0), (8192, 32, 256, 64, 1), (16896, 131, 64, 128, 0), (33792, 64, 128, 256, 0),
    # more units than SMs on 64- and 128-wide tiles
    (17025, 32, 64, 1, 1), (17023, 131, 128, 1, 0),
]
MLP_GROUPED = (4223, 99, 128, 1, 0, 103)                                       # 41 groups of 103 rows, across the tiles


def test_mlp_cases_cover_both_tile_widths_past_one_wave():
    seen = {Mlp(*c[:4]).plan()["Nt"] for c in MLP if Mlp(*c[:4]).plan()["units"] > R.PLAN_SMS}
    assert seen == {64, 128}


@pytest.mark.parametrize("case", MLP + [MLP_GROUPED], ids=lambda c: "x".join(map(str, c)))
@pytest.mark.parametrize("mode", (0, 2))
def test_shared_mlp_dense_layer_matches_float64(case, mode):
    """the dense op on the ring: its producer stages rows by 16- or 4-byte copies into stale shared memory, its consumers mask the
    rows past the end and the columns past K, and its epilogue stores, pools or takes the ordered-int max"""
    rows, K, N, pool_k, offset = case[:5]
    op = Mlp(rows, K, N, pool_k, offset, group_rows=case[5] if len(case) > 5 else 0, seed=rows + K)
    _check(op, mode)
