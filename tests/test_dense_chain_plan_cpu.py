"""The workspace plans of the inference dense layers, restated in tests/restate.py, against the library's size queries and
psa_mlp_image_plan in modes 0, 1 and 2: the chain of psa_shared_mlp / psa_sa_group_all_infer, the set-abstraction level and
EdgeConv.  No GPU needed."""
import ctypes as C
import itertools
import random

import pytest

from scanobjectnn_b200 import _lib

from . import restate as R

ROWS = (1, 32, 33, 127, 128, 4096)
WIDTHS = (15, 63, 64, 99, 128, 192, 256, 512, 1024)
USAGE_SHARED_MLP, USAGE_SA_GROUP_ALL, USAGE_SA_MODULE = 0, 1, 2


@pytest.fixture(params=[0, 1, 2], ids=["fp16x2", "fma", "bf16x3"])
def mode(request):
    lib = _lib.load()
    assert lib.psa_set_mlp_mode(request.param) == 0
    yield request.param
    lib.psa_set_mlp_mode(0)


def mlp_struct(channels):
    """a psa_mlp of these widths whose pointers are never dereferenced: the queries read the shapes only"""
    m = _lib.PsaMlp()
    m.n_layers = len(channels) - 1
    for l, ch in enumerate(channels):
        m.channels[l] = ch
    for l in range(m.n_layers):
        m.weight[l] = m.shift[l] = 16
    return m


def mlps():
    """every one-layer MLP of the widths, and a seeded sample of two to four layers"""
    rng = random.Random(7)
    out = [list(p) for p in itertools.product(WIDTHS, repeat=2)]
    for L in (2, 3, 4):
        out += [[rng.choice(WIDTHS) for _ in range(L + 1)] for _ in range(60)]
    return out


def image_plan(lib, usage, rows, pool_k, c, nsample, m):
    nt, row0, nbytes = (C.c_int * 4)(), (C.c_int * 4)(), (C.c_size_t * 4)()
    assert lib.psa_mlp_image_plan(usage, rows, pool_k, c, nsample, C.byref(m), nt, row0, nbytes) == 0
    return [(nt[l], row0[l], nbytes[l]) for l in range(4)]


def padded(entries):
    return entries + [(0, 0, 0)] * (4 - len(entries))


def test_chain_workspace_and_images_match_the_plan(mode):
    lib = _lib.load()
    for ch, rows in itertools.product(mlps(), ROWS):
        m = mlp_struct(ch)
        assert lib.psa_shared_mlp_workspace_bytes(rows, C.byref(m)) == R.chain_plan(rows, ch, ch[0])["total"], (ch, rows)
        for pool_k in {1, 32, rows}:
            want = [(0, 0, 0)] * 4 if mode == 1 else padded(R.chain_images(rows, pool_k, ch, 0, mode))
            assert image_plan(lib, USAGE_SHARED_MLP, rows, pool_k, 0, 0, m) == want, (ch, rows, pool_k)


def test_group_all_workspace_and_images_match_the_plan(mode):
    lib = _lib.load()
    for ch, (b, n) in itertools.product(mlps(), [(1, 1), (1, 32), (1, 33), (1, 127), (1, 128), (32, 128), (2, 2048)]):
        c = ch[0]
        gch = [3 + c] + ch[1:]
        m = mlp_struct(gch)
        assert lib.psa_sa_group_all_workspace_bytes(b, n, c, C.byref(m)) == R.chain_plan(b * n, gch, c)["total"], (ch, b, n)
        want = [(0, 0, 0)] * 4 if mode == 1 else padded(R.chain_images(b * n, n, gch, 3, mode))
        assert image_plan(lib, USAGE_SA_GROUP_ALL, b * n, n, 0, 0, m) == want, (ch, b, n)


def test_sa_module_workspace_and_images_match_the_plan(mode):
    lib = _lib.load()
    levels = [[64, 64, 128], [64, 128, 256], [128, 128, 256], [64, 64, 128, 1024], [128, 128, 128, 1024], [128, 128, 64, 512],
              [64, 128, 128, 2048], [128, 128, 128, 4096], [99, 64, 128], [64, 63, 128], [128, 64, 128, 192]]
    for (c, (b, n, m_, nsample)), lv in itertools.product(
            itertools.product((0, 3, 15, 64, 128, 320), [(1, 32, 8, 32), (2, 512, 128, 64), (8, 1024, 512, 32), (4, 128, 32, 128),
                                                         (1, 64, 16, 48)]), levels):
        ch = [3 + c] + lv
        m = mlp_struct(ch)
        layers = R.sa_tc_layers(ch, c, nsample, mode)
        want = 0 if layers is None else R.sa_workspace(b, n, c, ch, layers)
        assert lib.psa_sa_module_workspace_bytes(b, n, m_, c, nsample, C.byref(m)) == want, (ch, b, n, nsample)
        want = [(0, 0, 0)] * 4 if mode == 1 else R.sa_images(b * n, c, nsample, ch, mode)
        assert image_plan(lib, USAGE_SA_MODULE, b * n, 1, c, nsample, m) == want, (ch, b, n, nsample)


def test_edgeconv_workspace_matches_the_plan(mode):
    lib = _lib.load()
    tails = [[64], [128], [256], [32], [99], [512], [64, 128], [64, 128, 1024], [128, 64, 128], [64, 64, 4096]]
    for (b, n), c, k, tail in itertools.product([(1, 1), (1, 127), (1, 128), (8, 1024)], (1, 3, 15, 64), (1, 20, 32, 40), tails):
        ch = [2 * c] + tail
        m = mlp_struct(ch)
        assert lib.psa_edgeconv_workspace_bytes(b, n, c, k, C.byref(m)) == R.edgeconv_workspace(b, n, c, k, ch, mode), (b, n, c, k, ch)
