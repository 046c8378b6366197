"""The training entry points refuse, before any launch, the operands their vector loads or grids cannot take.  The pointers are fake
and never dereferenced: every call here fails its argument checks, so no test needs (or touches) a GPU."""
import ctypes as C

import pytest

from scanobjectnn_b200 import _lib
from scanobjectnn_b200._lib import PsaGradIn

A = 1 << 20                    # a fake 16-byte-aligned address; A + 4 is not
BIG = C.c_size_t(1 << 40)      # a workspace size that passes every size check


def _grad(mode, width, rows=None, pool_k=20):
    g = PsaGradIn(y=A, ld=width, s=A, t=A, relu=1, ca=A, cb=A, cc=A, C=width, mode=mode)
    if mode == 0:
        g.dh, g.ld_dh, g.mask = A, width, A
    else:
        g.dp, g.pv, g.argk, g.pool_k = A, A, A, pool_k
    return g


def _variants(width):
    """(name, grad_in, expected message fragment): each breaks one requirement of a valid mode-0 or mode-1 operand"""
    out = []
    for f in ("y", "s", "t", "ca", "cb", "cc", "dh", "mask"):
        g = _grad(0, width)
        setattr(g, f, A + 4)
        out.append((f"{f}+4", g, {"y": "y must", "s": "s / t", "t": "s / t", "dh": "dh / mask", "mask": "dh / mask"}.get(f, "ca / cb / cc")))
    g = _grad(0, width); g.ld = width + 2
    out.append(("ld%4", g, "y must"))
    g = _grad(0, width); g.ld_dh = width + 1
    out.append(("ld_dh%4", g, "ld_dh"))
    g = _grad(0, width); g.mode = 2
    out.append(("mode2", g, "mode"))
    for f in ("dp", "pv", "argk"):
        g = _grad(1, width)
        setattr(g, f, A + 4)
        out.append((f"{f}+4", g, "dp / pv / argk"))
    g = _grad(1, width); g.C = width + 4
    out.append(("C!=width", g, "pooled grad_in"))
    g = _grad(1, width, pool_k=7)
    out.append(("pool_k", g, "pooled grad_in"))
    return out


def _refused(lib, rc, frag, want=-1):
    msg = lib.psa_last_error().decode()
    assert rc == want and frag in msg, (rc, msg)


@pytest.mark.parametrize("entry", ["bn_bwd_coeffs", "sa_conv1_bwd", "sa_conv1_bwd_xyz"])
def test_reductions_refuse_operands_their_vector_loads_cannot_read(entry):
    lib = _lib.load()
    b, n, m, k, C1 = 2, 64, 16, 20, 64               # 640 grouped rows: pool_k 20 divides them, 7 does not
    rows = b * m * k
    p = C.c_void_p(A)
    for name, g, frag in _variants(C1):
        if entry == "bn_bwd_coeffs":
            if frag == "ca / cb / cc":
                continue                             # ignored there: the call computes them
            rc = lib.psa_bn_bwd_coeffs(rows, C1, C.byref(g), p, p, p, p, p, p, p, p, BIG, None)
        elif entry == "sa_conv1_bwd":
            rc = lib.psa_sa_conv1_bwd(b, n, m, k, C1, p, p, p, C.byref(g), p, p, p, BIG, None)
        else:
            rc = lib.psa_sa_conv1_bwd_xyz(b, n, m, k, C1, p, p, C.byref(g), p, p, p, BIG, None)
        _refused(lib, rc, frag)
        assert entry in lib.psa_last_error().decode(), name
    g = _grad(0, C1)
    rc = {"bn_bwd_coeffs": lambda: lib.psa_bn_bwd_coeffs(rows, C1, C.byref(g), p, C.c_void_p(A + 4), p, p, p, p, p, p, BIG, None),
          "sa_conv1_bwd": lambda: lib.psa_sa_conv1_bwd(b, n, m, k, C1, p, p, p, C.byref(g), p, C.c_void_p(A + 4), p, BIG, None),
          "sa_conv1_bwd_xyz": lambda: lib.psa_sa_conv1_bwd_xyz(b, n, m, k, C1, p, p, C.byref(g), p, p, C.c_void_p(A + 4), BIG, None)}[entry]()
    _refused(lib, rc, {"bn_bwd_coeffs": "mean_inv", "sa_conv1_bwd": "dU", "sa_conv1_bwd_xyz": "workspace"}[entry])


def test_pools_refuse_unaligned_operands():
    lib = _lib.load()
    for i in range(5):
        args = [C.c_void_p(A + (4 if j == i else 0)) for j in range(5)]
        _refused(lib, lib.psa_train_pool_fwd(10, 20, 64, *args, None), "16-byte aligned")
    for i in range(2):
        x, out = (C.c_void_p(A + (4 if j == i else 0)) for j in range(2))
        _refused(lib, lib.psa_pool_rows(10, 20, 64, 0, x, None, out, None), "16-byte aligned")


def test_row_tiles_beyond_the_grid_are_unsupported():
    """the fp32 GEMM puts 128-row tiles on gridDim.y: more than 65535 of them is refused up front"""
    lib = _lib.load()
    p = C.c_void_p(A)
    rows = 65536 * 128
    ain = _lib.PsaActIn(x=A, ld=64)
    g = PsaGradIn(dh=A, ld_dh=64, pool_k=1, C=64)
    _refused(lib, lib.psa_train_dense_fwd(rows, 64, 64, C.byref(ain), p, None, p, None, None, C.c_size_t(0), None), "row tiles", -2)
    _refused(lib, lib.psa_train_dense_fwd_grouped(rows, 128, 64, 64, C.byref(ain), p, None, p, p, None, None, C.c_size_t(0), None), "row tiles", -2)
    _refused(lib, lib.psa_train_dense_bwd_input(rows, 64, 64, C.byref(g), p, p, 64, 0, None, C.c_size_t(0), None), "row tiles", -2)
