"""The training GEMM (csrc/train_gemm.cuh, driven by csrc/train.cu) against float64 on each launch path and operand source: the
forward (tensor cores, small-M split, one fp32 pass), the grouped forward, the input gradient (split, its one-split fallback,
col_skip), the weight gradient (all four tilings, one and many splits), the bias and batch-norm sums and the max-pool routing.

Operands are restated from include/psa.h's psa_act_in / psa_grad_in in float64 torch.  Errors are relative to the largest entry
(restate.rel); the bounds are those of tests/test_train_gpu.py for the same kind of product, or, for a contraction too long for fp32
to meet them, 3x the error of the same product evaluated in float32 by torch (TF32 off).  Values that decide a relu gate or a max
(y, s, t of a psa_grad_in) lie on a dyadic grid, so fp32 and float64 take the same decisions, ties included.  Every dense call
gets exactly psa_train_dense_workspace_bytes, NaN-filled, with a NaN canary behind it, and runs twice: bit-identical results.
tests/test_train_gemm_plan_cpu.py checks that the cases reach every path."""
import ctypes as C

import numpy as np
import pytest
import torch

from scanobjectnn_b200 import _lib
from scanobjectnn_b200._lib import PsaActIn, PsaGradIn, ptr, stream

from . import restate as R

pytestmark = pytest.mark.gpu

TOL_Y, TOL_DX, TOL_DW, TOL_TC = 2e-6, 2e-6, 5e-6, 1e-5
TOL_SUM = 1e-5                 # bias and batch-norm sums: ten times tighter than tests/test_train_gpu.py's 1e-4 for the latter
CANARY = 64                    # floats behind the queried workspace
F64, F32 = torch.float64, torch.float32


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _normal(shape, g, scale=1.0):
    return torch.randn(shape, generator=g, device="cuda") * scale


def _dyadic(shape, g, lo, hi, den):
    return torch.randint(lo, hi + 1, shape, generator=g, device="cuda").float() / den


def _check(what, got, want, want32, tol):
    e, e32 = R.rel(got.cpu().numpy(), want.cpu().numpy()), R.rel(want32.cpu().numpy(), want.cpu().numpy())
    print(f"{what}: err {e:.2e}  float32 {e32:.2e}  bound {tol:.0e} or 3x float32")
    assert R.within(e, e32, tol, 3.0), (what, e, e32)


class Workspace:
    """exactly the queried bytes, NaN-filled, and a NaN canary behind them"""

    def __init__(self, lib, rows, K, N):
        self.need = lib.psa_train_dense_workspace_bytes(rows, K, N)
        assert self.need % 4 == 0
        self.buf = torch.full((self.need // 4 + CANARY,), float("nan"), device="cuda")

    def args(self):
        return ptr(self.buf), C.c_size_t(self.need)

    def check(self):
        assert torch.isnan(self.buf[self.need // 4:]).all(), "a write past the queried workspace"

    def written(self, count):
        return not torch.isnan(self.buf[:count]).any()


def _layout(rows, K, x_layout, g, fill):
    """a (rows, K) view of `fill`ed storage in the given layout, and its ld"""
    if x_layout == "dense":
        return fill((rows, K), g), K
    if x_layout == "slice":
        return fill((rows, K + 8), g)[:, 8:], K + 8
    if x_layout == "ld_odd":
        return fill((rows, K + 3), g)[:, :K], K + 3
    assert x_layout == "offset"
    return fill((rows * K + 1,), g)[1:].view(rows, K), K


def act_in(rows, K, act, x_layout, g):
    """(psa_act_in, tensors to keep alive, h in float64, h in float32)"""
    x, ld = _layout(rows, K, x_layout, g, lambda s, g: _normal(s, g))
    keep = [x]
    a = PsaActIn(x=x.data_ptr(), ld=ld)
    h64, h32 = x.double(), x.clone()
    if act != "raw":
        off = 1 if x_layout == "offset" else 0
        s = (torch.rand(K + off, generator=g, device="cuda") + 0.5)[off:]
        t = _normal(K + off, g, 0.3)[off:]
        keep += [s, t]
        a.scale, a.shift, a.relu = s.data_ptr(), t.data_ptr(), 1
        h64 = torch.clamp_min(h64 * s.double() + t.double(), 0)
        h32 = torch.clamp_min(torch.addcmul(t, h32, s), 0)
    if act == "bn_mask":
        m, _ = _layout(rows, K, x_layout, g, lambda s, g: (torch.rand(s, generator=g, device="cuda") < 0.5).float() * 2)
        keep.append(m)
        a.mask = m.data_ptr()
        h64, h32 = h64 * m.double(), h32 * m
    return a, keep, h64, h32


def pool_routing(lib, y, s, t, pool_k):
    """psa_train_pool_fwd on y, checked exactly: relu(y * s + t) is exact on the dyadic grid, argk the first winning row and a
    group that is all <= 0 pools 0 with argk 0"""
    rows, N = y.shape
    G = rows // pool_k
    pooled = torch.empty((G, N), device="cuda")
    argk = torch.empty((G, N), dtype=torch.int32, device="cuda")
    assert lib.psa_train_pool_fwd(G, pool_k, N, ptr(y), ptr(s), ptr(t), ptr(pooled), ptr(argk), stream()) == 0
    z = torch.clamp_min(y.double() * s.double() + t.double(), 0).view(G, pool_k, N)
    want_p, _ = z.max(1)
    want_k = (z == want_p[:, None, :]).int().argmax(1)          # the first row that reaches the max
    assert torch.equal(pooled.double(), want_p) and torch.equal(argk.long(), want_k.long())
    zero = want_p == 0
    assert zero.any() and (~zero).any() and ((z == want_p[:, None, :]).sum(1) > 1).any(), "want ties and empty groups"
    return pooled, argk


def grad_in(lib, rows, N, src, g):
    """(psa_grad_in, tensors to keep alive, dy in float64, dy in float32) for the '+'-joined flags of `src`"""
    flags = set(src.split("+"))
    pool_k = 20 if "pool20" in flags else 32 if "pool32" in flags else 0
    ld = N + 3 if "scalar" in flags else N
    ybuf = _dyadic((rows, ld), g, -6, 6, 4)
    y = ybuf[:, :N]
    s, t = 1 + _dyadic((N,), g, -2, 2, 8), _dyadic((N,), g, -4, 4, 8)
    keep = [ybuf, s, t]
    gi = PsaGradIn(y=y.data_ptr(), ld=ld, C=N, pool_k=max(pool_k, 1))
    gate = ((y.double() * s.double() + t.double()) > 0).double()
    if pool_k:
        G = rows // pool_k
        y.view(G, pool_k, N)[0] = -4                                  # a group that is all <= 0 after batch norm and relu
        y.view(G, pool_k, N)[1, :, : N // 2] = -4
        pooled, argk = pool_routing(lib, y, s, t, pool_k)
        dp = _normal((G, N), g)
        keep += [pooled, argk, dp]
        gi.mode, gi.dp, gi.pv, gi.argk = 1, dp.data_ptr(), pooled.data_ptr(), argk.data_ptr()
        gi.s, gi.t, gi.relu = s.data_ptr(), t.data_ptr(), 1           # mode 1 ignores the gate: pv > 0 is the relu
        dz = torch.zeros((G, pool_k, N), dtype=F64, device="cuda")
        win = (pooled > 0).double() * dp.double()
        dz.scatter_(1, argk.long()[:, None, :], win[:, None, :])
        dz64 = dz.view(rows, N)
    else:
        ld_dh = N + 1 if "scalar" in flags else N
        dh = _normal((rows, ld_dh), g)
        keep.append(dh)
        gi.dh, gi.ld_dh = dh.data_ptr(), ld_dh
        dz64 = dh[:, :N].double()
        if "mask" in flags:
            m = (torch.rand((rows, ld_dh), generator=g, device="cuda") < 0.5).float() * 2
            keep.append(m)
            gi.mask = m.data_ptr()
            dz64 = dz64 * m[:, :N].double()
        if "gate" in flags:
            gi.s, gi.t, gi.relu = s.data_ptr(), t.data_ptr(), 1
            dz64 = dz64 * gate
    dz32 = dz64.float()
    dy64, dy32 = dz64, dz32
    if "coeffs" in flags:
        ca, cb, cc = _normal(N, g), _normal(N, g, 0.1), _normal(N, g, 0.1)
        keep += [ca, cb, cc]
        gi.ca, gi.cb, gi.cc = ca.data_ptr(), cb.data_ptr(), cc.data_ptr()
        dy64 = ca.double() * dz64 + cb.double() * y.double() + cc.double()
        dy32 = torch.addcmul(torch.addcmul(cc, cb, y), ca, dz32)
    return gi, keep, dy64, dy32


def _twice(call, out):
    """run `call` twice: the second result must be bit-identical to the first"""
    assert call() == 0, _lib.load().psa_last_error()
    first = out.clone()
    out.fill_(float("nan"))
    assert call() == 0
    assert torch.equal(first.view(torch.int32), out.view(torch.int32)), "not bit-reproducible"
    return first


@pytest.mark.parametrize("case", R.FWD_CASES, ids=[c[0] for c in R.FWD_CASES])
def test_forward(case):
    name, rows, K, N, act, x_layout, use_bias, use_stats = case
    lib = _lib.load()
    g = _gen(rows * 7 + K)
    a, keep, h64, h32 = act_in(rows, K, act, x_layout, g)
    W = _normal((K, N), g, K ** -0.5)
    b = _normal(N, g, 0.1) if use_bias else None
    y = torch.empty((rows, N), device="cuda")
    stats = torch.empty((2, N), device="cuda") if use_stats else None
    ws = Workspace(lib, rows, K, N)
    plan = R.train_fwd_plan(rows, K, N, ld=a.ld, mask=act == "bn_mask")
    got = _twice(lambda: lib.psa_train_dense_fwd(rows, K, N, C.byref(a), ptr(W), ptr(b), ptr(y), ptr(stats), *ws.args(), stream()), y)
    want, want32 = h64 @ W.double(), h32 @ W
    if b is not None:
        want, want32 = want + b.double(), want32 + b
    _check(f"{name} ({plan['path']}) y", got, want, want32, TOL_TC if plan["path"] == "tc" else TOL_Y)
    if use_stats:
        _check_stats(stats, want)
    ws.check()


def _check_stats(stats, y):
    """column sums and sums of squares, as tests/test_train_gpu.py checks them"""
    st, w = stats.double().cpu().numpy(), y.cpu().numpy()
    np.testing.assert_allclose(st[0], w.sum(0), rtol=1e-5, atol=1e-3 * np.sqrt(len(w)))
    np.testing.assert_allclose(st[1], (w ** 2).sum(0), rtol=1e-5, atol=1e-3)


@pytest.mark.parametrize("rows,group_rows,K,N", [(300, 50, 40, 48), (519, 173, 70, 96)])
def test_grouped_forward(rows, group_rows, K, N):
    """group rows not aligned to the 128-row tiles, bias, statistics, an input with batch norm, relu and dropout"""
    lib = _lib.load()
    g = _gen(rows + group_rows)
    a, keep, h64, h32 = act_in(rows, K, "bn_mask", "dense", g)
    W, b = _normal((K, N), g, K ** -0.5), _normal(N, g, 0.1)
    ga = _normal((rows // group_rows, N), g)
    y, stats = torch.empty((rows, N), device="cuda"), torch.empty((2, N), device="cuda")
    ws = Workspace(lib, rows, K, N)
    got = _twice(lambda: lib.psa_train_dense_fwd_grouped(rows, group_rows, K, N, C.byref(a), ptr(W), ptr(b), ptr(ga), ptr(y), ptr(stats),
                                                         *ws.args(), stream()), y)
    rep = torch.arange(rows, device="cuda") // group_rows
    want = h64 @ W.double() + ga.double()[rep] + b.double()
    _check(f"grouped {rows}/{group_rows} y", got, want, h32 @ W + ga[rep] + b, TOL_Y)
    _check_stats(stats, want)
    ws.check()


@pytest.mark.parametrize("case", R.BWD_INPUT_CASES, ids=[c[0] for c in R.BWD_INPUT_CASES])
def test_input_gradient(case):
    name, rows, K, N, src, col_skip, ld_dx = case
    lib = _lib.load()
    g = _gen(rows * 3 + N)
    gi, keep, dy64, dy32 = grad_in(lib, rows, N, src, g)
    W = _normal((K, N), g, N ** -0.5)
    width = K - col_skip
    ld_dx = ld_dx or width
    dxbuf = torch.full((rows, ld_dx), float("nan"), device="cuda")
    dx = dxbuf[:, :width]
    ws = Workspace(lib, rows, K, N)
    plan = R.train_bwd_input_plan(rows, K, N, ws.need)
    want, want32 = (dy64 @ W.double().T)[:, col_skip:], (dy32 @ W.T)[:, col_skip:]
    got = _twice(lambda: lib.psa_train_dense_bwd_input(rows, K, N, C.byref(gi), ptr(W), ptr(dx), ld_dx, col_skip, *ws.args(), stream()), dxbuf)
    _check(f"{name} ({plan['path']}) dx", got[:, :width], want, want32, TOL_DX)
    assert torch.isnan(got[:, width:]).all(), "a write past the dx view"
    ws.check()
    # the split path writes its partials into the workspace; without one it runs a single split and must agree
    assert ws.written(plan["splits"] * rows * K) == (plan["path"] == "split")
    if plan["path"] == "split":
        got1 = _twice(lambda: lib.psa_train_dense_bwd_input(rows, K, N, C.byref(gi), ptr(W), ptr(dx), ld_dx, col_skip, None, C.c_size_t(0),
                                                            stream()), dxbuf)
        _check(f"{name} (one split, no workspace) dx", got1[:, :width], want, want32, TOL_DX)
        e = R.rel(got1[:, :width].cpu().numpy(), got[:, :width].double().cpu().numpy())
        print(f"{name}: split vs one split {e:.2e}")
        assert e < TOL_DX


@pytest.mark.parametrize("case", R.BWD_WEIGHT_CASES, ids=[c[0] for c in R.BWD_WEIGHT_CASES])
def test_weight_gradient(case):
    name, rows, K, N, act, x_layout, src = case
    lib = _lib.load()
    g = _gen(rows * 5 + K * N)
    a, keep_a, h64, h32 = act_in(rows, K, act, x_layout, g)
    gi, keep_g, dy64, dy32 = grad_in(lib, rows, N, src, g)
    dW = torch.empty((K, N), device="cuda")
    ws = Workspace(lib, rows, K, N)
    plan = R.train_bwd_weight_plan(rows, K, N)
    got = _twice(lambda: lib.psa_train_dense_bwd_weight(rows, K, N, C.byref(a), C.byref(gi), ptr(dW), *ws.args(), stream()), dW)
    _check(f"{name} ({plan['bm']}x{plan['bn']}, {plan['splits']} splits) dW", got, h64.T @ dy64, h32.T @ dy32, TOL_DW)
    ws.check()
    assert ws.written(plan["splits"] * K * N) == (plan["splits"] > 1)


BIAS_SRCS = ["plain", "mask", "gate", "coeffs", "mask+gate+coeffs", "pool20", "pool32+coeffs", "scalar+mask+gate+coeffs"]


@pytest.mark.parametrize("src", BIAS_SRCS)
def test_bias_gradient(src):
    """psa_train_bias_grad and _grouped (groups of 64 rows, not aligned to the 256-thread blocks' strides) from every source"""
    lib = _lib.load()
    rows, N = 1280, 68
    g = _gen(len(src))
    gi, keep, dy64, dy32 = grad_in(lib, rows, N, src, g)
    db = torch.empty(N, device="cuda")
    got = _twice(lambda: lib.psa_train_bias_grad(rows, N, C.byref(gi), ptr(db), stream()), db)
    _check(f"bias {src}", got, dy64.sum(0), dy32.sum(0), TOL_SUM)
    G = rows // 64
    dbg = torch.empty((G, N), device="cuda")
    got = _twice(lambda: lib.psa_train_bias_grad_grouped(rows, 64, N, C.byref(gi), ptr(dbg), stream()), dbg)
    _check(f"bias grouped {src}", got, dy64.view(G, 64, N).sum(1), dy32.view(G, 64, N).sum(1), TOL_SUM)


@pytest.mark.parametrize("rows,Cc,src", [(1_200_000, 4, "mask+gate"), (400_000, 12, "mask+gate"), (5000, 1024, "mask+gate"),
                                         (3000, 64, "plain"), (2000, 64, "pool20"), (4096, 128, "pool32")])
def test_bn_backward_sums(rows, Cc, src):
    """psa_bn_bwd_coeffs: dbeta = sum dz, dgamma = sum dz * (y - mean) * inv, and the coefficients from them.  The first three shapes
    hit the kBnbMaxBlocks cap of the partial blocks; "plain" has no relu gate (s = NULL), where y is still read for xhat."""
    lib = _lib.load()
    g = _gen(rows + Cc)
    gi, keep, dy64, _ = grad_in(lib, rows, Cc, src, g)
    yv = keep[0].double()                                                 # y, after grad_in's changes for the pooled cases
    mean = yv.mean(0).float()
    inv = (1 / torch.sqrt(yv.var(0, unbiased=False) + 1e-3)).float()
    mean_inv = torch.stack([mean, inv])
    gamma = torch.rand(Cc, generator=g, device="cuda") + 0.5
    dgamma, dbeta, ca, cb, cc = (torch.empty(Cc, device="cuda") for _ in range(5))
    need = lib.psa_bn_bwd_workspace_bytes(Cc)
    wsb = torch.full((need // 4 + CANARY,), float("nan"), device="cuda")
    out = torch.empty((5, Cc), device="cuda")

    def call():
        rc = lib.psa_bn_bwd_coeffs(rows, Cc, C.byref(gi), ptr(gamma), ptr(mean_inv), ptr(dgamma), ptr(dbeta), ptr(ca), ptr(cb), ptr(cc),
                                   ptr(wsb), C.c_size_t(need), stream())
        torch.stack([dgamma, dbeta, ca, cb, cc], out=out)
        return rc

    got = _twice(call, out).double()
    assert torch.isnan(wsb[need // 4:]).all()
    dz = dy64                                                             # no coefficients in src: dy is dz
    xhat = (yv - mean.double()) * inv.double()
    db, dg = dz.sum(0), (dz * xhat).sum(0)
    gm, mu, iv = gamma.double(), mean.double(), inv.double()
    want = [dg, db, gm * iv, -gm * iv * iv * dg / rows, gm * iv * (mu * iv * dg - db) / rows]
    for what, got_i, want_i in zip(("dgamma", "dbeta", "ca", "cb", "cc"), got, want):
        e = R.rel(got_i.cpu().numpy(), want_i.cpu().numpy())
        print(f"bn {rows}x{Cc} {src} {what}: err {e:.2e}  bound {TOL_SUM:.0e}")
        assert e < TOL_SUM, (what, e)
