"""conv_wgrad_tc_kernel over grids with several 128-channel output tiles, which the instance table of conv_cases.py
reaches only with two: 2, 3, 4 and 8 tiles, a short last tile whose second warpgroup has no channels (Cout 192, 448), the
three box widths, stride 2 with odd sizes, one and many pixel tiles per split, a single split of several tiles that adds
into dw, and the fully-connected layers at the box head's (256, 49) feature order.  Each result is checked against
float64 inside guarded buffers and recomputed with equal bits."""
import math

import pytest
import torch

import conv_cases as cc
from test_conv_dispatch_gpu import Guarded, _bf, _gen, _lin_x, _nchw, _randn

pytestmark = pytest.mark.gpu

COTILE_CASES = [
    cc._case(Cin=256, Cout=256, k=3, H=20, W=24),              # 2 co tiles, cw 64: one 5-D x box of 4 chunks per stage
    cc._case(Cin=64, Cout=192, k=3, H=10, W=14),               # 2 co tiles, the last one 64 channels: idle second warpgroup
    cc._case(Cin=64, Cout=320, k=1, H=10, W=14),               # 3 co tiles
    cc._case(Cin=96, Cout=448, k=1, N=3, H=20, W=24),          # 4 co tiles, short last; cw 32, three x loads per stage
    cc._case(Cin=16, Cout=512, k=3, s=2, H=27, W=31),          # 4 co tiles, cw 16, nine x loads; stride 2, odd sizes
    cc._case(Cin=32, Cout=1024, k=1, N=1, H=9, W=9),           # 8 co tiles, one tile per split, a single x box
    cc._case(Cin=128, Cout=256, k=3, N=8, H=40, W=40),         # many splits of many tiles, last column group 2 boxes
    cc._case(Cin=256, Cout=1024, k=3, N=1, H=16, W=24),        # 72 CTAs per split: one split of three tiles adds into dw
]


def _co_tiles(Cout):
    return -(-Cout // 128)


@pytest.mark.parametrize("c", COTILE_CASES, ids=cc.case_id)
def test_wgrad_co_tiles(c):
    """OHWI into zeros (twice: equal bits), then OIHW added to a pre-loaded gradient"""
    from omni3d_b200 import conv as K
    inst, buckets, single = cc.wgrad_plan(cc.fwd_desc(c))
    assert inst[0] == "gemm"
    name = (f"wgrad {cc.case_id(c)} {inst} co tiles {_co_tiles(c.Cout)} ncols {sorted(buckets)} "
            f"{'one split' if single else 'splits'}")
    g = _gen(16)
    Ho, Wo = cc.out_size(cc.fwd_desc(c))
    x = _bf(_randn(g, c.N, c.H, c.W, c.Cin))
    dy = _bf(_randn(g, c.N, Ho, Wo, c.Cout))
    wsize = (c.Cout, c.Cin, c.k, c.k)
    r = torch.nn.grad.conv2d_weight(_nchw(x), wsize, _nchw(dy), c.s, c.p)
    A = torch.nn.grad.conv2d_weight(_nchw(x).abs(), wsize, _nchw(dy).abs(), c.s, c.p)
    n = math.prod(wsize)
    G = Guarded(n, torch.float32)
    dw = G.mark(G.view((c.Cout, c.k, c.k, c.Cin))).zero_()
    K.conv2d_wgrad(x, dy, c.k, c.k, c.s, c.p, dw=dw, oihw=False)
    dw2 = K.conv2d_wgrad(x, dy, c.k, c.k, c.s, c.p, oihw=False)
    torch.cuda.synchronize()
    cc.check(name + " ohwi", dw, r.permute(0, 2, 3, 1), A.permute(0, 2, 3, 1), 0.0, cc.GAMMA_WGRAD)
    G.check(name + " ohwi")
    assert torch.equal(dw.view(torch.int32), dw2.view(torch.int32)), f"{name}: second call differs"
    G = Guarded(n, torch.float32)
    dwo = G.mark(G.view(wsize))
    dw_in = _randn(g, *wsize, scale=r.abs().max().item())
    dwo.copy_(dw_in)
    K.conv2d_wgrad(x, dy, c.k, c.k, c.s, c.p, dw=dwo, oihw=True)
    torch.cuda.synchronize()
    cc.check(name + " oihw", dwo, r + dw_in.double(), A + dw_in.double().abs(), 0.0, cc.GAMMA_WGRAD)
    G.check(name + " oihw")


def test_cases_cover_the_grids():
    """the table above reaches even and odd tile counts, every box width, a single split and many"""
    plans = [(c, cc.wgrad_plan(cc.fwd_desc(c))) for c in COTILE_CASES]
    assert {_co_tiles(c.Cout) for c, _ in plans} >= {2, 3, 4, 8}
    assert {p[0][1] for c, p in plans if _co_tiles(c.Cout) % 2 == 0} == set(cc.WGRAD_WIDTHS)
    assert {p[2] for c, p in plans if _co_tiles(c.Cout) % 2 == 0} == {True, False}


COTILE_LINEAR = [
    cc._lin(256 * 49, 256, 3, 100, 112, chw=(256, 49)),        # the box head's first layer order; 2 co tiles, row blocks
    cc._lin(1024, 1024, 1, 300, 300),                          # 8 co tiles, three splits
    cc._lin(64, 256, 3, 200, 230, chw=(16, 4)),                # cw 16, row blocks
]


@pytest.mark.parametrize("c", COTILE_LINEAR, ids=cc.lin_id)
def test_linear_wgrad_co_tiles(c):
    from omni3d_b200 import conv as K
    C, PP = c.chw if c.chw else (c.K, 1)
    inst, buckets, single = cc.wgrad_plan(cc.linear_descs(c)[0], C, PP)
    name = f"linear wgrad {cc.lin_id(c)} ({inst}, ncols {sorted(buckets)})"
    g = _gen(19)
    Gx, xall, xs = _lin_x(c, g)
    dy = _bf(_randn(g, c.nseg * c.rows, c.N))
    r = dy.double().T @ xs.double()                          # (N, K) in x's (p, c) feature order
    A = dy.double().abs().T @ xs.double().abs()
    r, A = (t.view(c.N, PP, C).transpose(1, 2).reshape(c.N, c.K) for t in (r, A))   # the master's (c, p) order
    dw_in = _randn(g, c.N, c.K, scale=r.abs().max().item())
    outs = []
    for _ in range(2):
        G = Guarded(c.N * c.K, torch.float32)
        dw = G.mark(G.view((c.N, c.K)))
        dw.copy_(dw_in)
        K.linear_wgrad(xall, dy, dw=dw, chw=c.chw, blocks=(c.nseg, c.rows, c.stride))
        torch.cuda.synchronize()
        cc.check(name, dw, r + dw_in.double(), A + dw_in.double().abs(), 0.0, cc.GAMMA_WGRAD)
        G.check(name)
        outs.append(dw.view(torch.int32).clone())
    Gx.check(name + " x")
    assert torch.equal(outs[0], outs[1]), f"{name}: second call differs"
