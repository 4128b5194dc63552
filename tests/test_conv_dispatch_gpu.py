"""Every compiled instance of the wgmma convolution (forward GEMM tiles, thin-channel halo kernels, weight-gradient tiles)
and every data-gradient route, against float64 references of the bf16 operands as stored, per element:
    |got - r| <= q*|r| + gamma*A           (conv_cases.check; A = the same operation on |operands|)
Outputs and strided inputs live inside allocations pre-filled with a NaN bit pattern: a store outside the described
tensor changes a guard, a read outside it turns an output into NaN.  The case table and the mirror of the selection
rules are in conv_cases.py; test_conv_dispatch_cpu.py asserts that the cases reach every instance."""
import math

import pytest
import torch
import torch.nn.functional as F

import conv_cases as cc

pytestmark = pytest.mark.gpu

PAD = 64                                         # guard elements before and after every allocation
SENTINEL = {torch.bfloat16: (torch.int16, 0x7FA5), torch.float32: (torch.int32, 0x7FA5A5A5)}   # NaN payloads


class Guarded:
    """a flat allocation filled with a NaN bit pattern.  The tensors a kernel reads or writes are views of it; every
    element no view was marked written must keep the pattern."""

    def __init__(self, numel, dtype):
        self.flat = torch.empty(numel + 2 * PAD, dtype=dtype, device="cuda")
        itype, self.sent = SENTINEL[dtype]
        self.bits = self.flat.view(itype)
        self.bits.fill_(self.sent)
        self.written = torch.zeros(self.flat.numel(), dtype=torch.bool, device="cuda")

    def view(self, shape, offset=0):
        return self.flat[PAD + offset:PAD + offset + math.prod(shape)].view(shape)

    def mark(self, v):
        torch.as_strided(self.written, v.size(), v.stride(), v.storage_offset()).fill_(True)
        return v

    def check(self, name):
        bad = (self.bits != self.sent) & ~self.written
        assert not bad.any(), (f"{name}: {int(bad.sum())} guard elements overwritten, first at flat index "
                               f"{(torch.nonzero(bad)[:4].flatten() - PAD).tolist()}")


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device="cuda") * scale


def _bf(t):
    return t.bfloat16()


def _master(g, Cout, Cin, k):
    """fp32 OIHW weight whose values are bf16-representable (the kernels' packs are then exact)"""
    return (_randn(g, Cout, Cin, k, k) / math.sqrt(Cin * k * k)).bfloat16().float()


def _ohwi(w):
    return w.permute(0, 2, 3, 1).contiguous().bfloat16()


def _nchw(t):
    return t.double().permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def conv_ref(x, w, c):
    """float64 (r, A) NHWC of the convolution the case describes (out_hw: zero padding on the high side)"""
    xd, wd = _nchw(x), w.double()
    if c.out_hw is None:
        f = lambda a, b: F.conv2d(a, b, stride=c.s, padding=c.p)
    else:
        Ho, Wo = c.out_hw
        f = lambda a, b: F.conv2d(F.pad(a, (c.p, c.p + c.s * Wo, c.p, c.p + c.s * Ho)), b, stride=c.s)[:, :, :Ho, :Wo]
    return _nhwc(f(xd, wd)), _nhwc(f(xd.abs(), wd.abs()))


def _check(name, got, r, A, fp32=False, gamma=cc.GAMMA_FWD):
    return cc.check(name, got, r, A, 0.0 if fp32 else cc.Q_BF16, gamma)


def _tile_sum(v, TH, TW):
    """(N, Ho, Wo, C) -> (tiles, C) sums over the conv_tc_kernel output tiles, in its tile order"""
    N, Ho, Wo, C = v.shape
    th, tw = -(-Ho // TH), -(-Wo // TW)
    v = F.pad(v, (0, 0, 0, tw * TW - Wo, 0, th * TH - Ho))
    return v.reshape(N, th, TH, tw, TW, C).sum((2, 4)).reshape(N * th * tw, C)


def _check_stats(name, stats, d, r, A, halo):
    """BatchNorm partial statistics of the raw accumulators: (sum, sum of squares) per output tile, or (halo kernel:
    one row per persistent CTA) their column totals.  Bound: the outputs' gamma*A per element, plus 2^-16 of the
    summed magnitudes for the fp32 sums."""
    from omni3d_b200 import conv as K
    tiles, TH, TW = K.num_tiles(d)
    assert stats.shape[0] == tiles, (name, tuple(stats.shape), tiles)
    e = cc.GAMMA_FWD * A
    parts = [(r, e + 2.0 ** -16 * r.abs()), (r * r, 2 * r.abs() * e + e * e + 2.0 ** -16 * r * r)]
    for which, (v, b) in enumerate(parts):
        if halo:
            got, ref, bnd = stats[:, which].double().sum(0), v.sum((0, 1, 2)), b.sum((0, 1, 2))
        else:
            assert tiles == r.shape[0] * -(-r.shape[1] // TH) * -(-r.shape[2] // TW), (name, tiles, TH, TW)
            got, ref, bnd = stats[:, which], _tile_sum(v, TH, TW), _tile_sum(b, TH, TW)
        worst = cc.worst_ratio(got, ref, bnd)
        print(f"{name} stats[{which}]: worst err/bound {worst:.3g}")
        assert worst <= 1.0, (name, which, worst)


def _fwd_desc(x, wp, c, relu, fp32, add_mode):
    from omni3d_b200 import conv as K
    d = K.make_desc(x, wp, c.s, c.p, relu, fp32, add_mode)
    if c.out_hw is not None:
        d.out_h, d.out_w = c.out_hw
    return d


def run_fwd(c, variant, seed):
    from omni3d_b200 import conv as K
    name = f"fwd {cc.case_id(c)} {variant}"
    g = _gen(seed)
    x = _bf(_randn(g, c.N, c.H, c.W, c.Cin))
    w = _master(g, c.Cout, c.Cin, c.k)
    b = _randn(g, c.Cout, scale=0.5)
    wp = _ohwi(w)
    r0, A0 = conv_ref(x, w, c)
    N, Ho, Wo, Co = r0.shape
    fp32 = variant == "fp32"
    relu = variant not in ("fp32", "acc_dense", "acc_slice")
    stats = variant in ("bias_relu_stats", "stats")
    acc = variant.startswith("acc")
    add_mode = {"addend": 1, "up2": 2, "acc_dense": 3, "acc_slice": 3}.get(variant, 0)
    r, A = r0 + b.double(), A0 + b.abs().double()
    dt = torch.float32 if fp32 else torch.bfloat16
    if variant in ("slice", "acc_slice"):        # channels [8, 8 + Cout) of a wider NHWC buffer
        G = Guarded(N * Ho * Wo * (Co + 24), dt)
        out = G.mark(G.view((N, Ho, Wo, Co + 24))[..., 8:8 + Co])
    else:
        G = Guarded(N * Ho * Wo * Co, dt)
        out = G.mark(G.view((N, Ho, Wo, Co)))
    addend = None
    if add_mode == 1:
        addend = _bf(_randn(g, N, Ho, Wo, Co))
        r, A = r + addend.double(), A + addend.double().abs()
    elif add_mode == 2:
        addend = _bf(_randn(g, N, Ho // 2, Wo // 2, Co))
        up = addend.double().repeat_interleave(2, 1).repeat_interleave(2, 2)
        r, A = r + up, A + up.abs()
    elif acc:
        prior = _bf(_randn(g, N, Ho, Wo, Co))
        out.copy_(prior)
        r, A = r + prior.double(), A + prior.double().abs()
    if relu:
        r = r.clamp_min(0)
    res = K.conv2d_fwd(x, wp, b, stride=c.s, pad=c.p, relu=relu, addend=addend, up2=add_mode == 2, out_fp32=fp32,
                       want_stats=stats, out=out, out_hw_override=c.out_hw, accumulate=acc)
    torch.cuda.synchronize()
    _check(name, out, r, A, fp32)
    G.check(name)
    if stats:
        d = _fwd_desc(x, wp, c, relu, fp32, add_mode)
        _check_stats(name, res[1], d, r0, A0, cc.fwd_instance(cc.fwd_desc(c))[0] == "halo")


@pytest.mark.parametrize("variant", cc.GEMM_VARIANTS)
@pytest.mark.parametrize("c", cc.GEMM_CASES, ids=cc.case_id)
def test_gemm_fwd_instances(c, variant):
    run_fwd(c, variant, seed=1)


@pytest.mark.parametrize("variant", cc.HALO_VARIANTS)
@pytest.mark.parametrize("c", cc.HALO_CASES, ids=cc.case_id)
def test_halo_fwd_instances(c, variant):
    run_fwd(c, variant, seed=2)


@pytest.mark.parametrize("c", cc.EDGE_CASES, ids=cc.case_id)
def test_fwd_edges(c):
    run_fwd(c, "bias_relu_stats", seed=3)


# ---- data gradient ---------------------------------------------------------------------------------------------------
def _dgrad_inputs(c, seed):
    g = _gen(seed)
    Ho, Wo = cc.out_size(cc.fwd_desc(c))
    dy = _bf(_randn(g, c.N, Ho, Wo, c.Cout))
    w = _master(g, c.Cout, c.Cin, c.k)
    size = (c.N, c.Cin, c.H, c.W)
    r = _nhwc(torch.nn.grad.conv2d_input(size, w.double(), _nchw(dy), c.s, c.p))
    A = _nhwc(torch.nn.grad.conv2d_input(size, w.double().abs(), _nchw(dy).abs(), c.s, c.p))
    return g, dy, w, r, A


@pytest.mark.parametrize("variant", cc.DGRAD_VARIANTS)
@pytest.mark.parametrize("c", cc.DGRAD_CASES, ids=cc.case_id)
def test_dgrad_routes(c, variant):
    """nnfunc._dgrad on a given dy (no ReLU mask): dense, added into a dense buffer, added into a channel slice"""
    from omni3d_b200 import nnfunc
    name = f"dgrad {cc.case_id(c)} {variant} ({cc.dgrad_route(c, variant == 'into_slice')})"
    g, dy, w, r, A = _dgrad_inputs(c, seed=4)
    shape = (c.N, c.H, c.W, c.Cin)
    if variant == "dense":
        dx = nnfunc._dgrad(dy, w, c.s, c.p, (c.H, c.W))
        torch.cuda.synchronize()
        _check(name, dx, r, A)
        return
    extra = 16 if variant == "into_slice" else 0
    G = Guarded(math.prod(shape) // c.Cin * (c.Cin + extra), torch.bfloat16)
    into = G.view(shape[:3] + (c.Cin + extra,))[..., extra // 2:extra // 2 + c.Cin]
    G.mark(into)
    prior = _bf(_randn(g, *shape))
    into.copy_(prior)
    dx = nnfunc._dgrad(dy, w, c.s, c.p, (c.H, c.W), into=into)
    torch.cuda.synchronize()
    assert dx is into
    _check(name, into, r + prior.double(), A + prior.double().abs())
    G.check(name)


_PHASE_CASES = [c for c in cc.DGRAD_CASES if cc.dgrad_route(c, False) in ("merged", "separate")]


@pytest.mark.parametrize("c", _PHASE_CASES, ids=cc.case_id)
def test_dgrad_phase_placement(c):
    """the stride-2 phase convolutions write exactly their parity positions of dx (y_img/h/w_stride, y_offset), and
    the merged 2x2 convolution exactly all of dx (y_split_c / y_split_off)"""
    from omni3d_b200 import conv as K
    from omni3d_b200 import nnfunc
    g, dy, w, r, A = _dgrad_inputs(c, seed=5)
    N, Ho, Wo, _ = dy.shape
    H, W, I = c.H, c.W, c.Cin
    packs = K.pack_conv_weight(w, phases=nnfunc._phase_layout(w))[2]
    for key, wp in packs.items():
        name = f"dgrad phase {cc.case_id(c)} {key}"
        G = Guarded(N * H * W * I, torch.bfloat16)
        dx = G.view((N, H, W, I))
        if key == "merged":
            K.conv2d_fwd(dy, wp, out=dx, out_place=(H * W, 2 * W, 2, 0), out_hw_override=(Ho, Wo),
                         split=(2 * I, W * I - 2 * I))
            sel = (slice(None),) * 3
        else:
            a, b = key
            K.conv2d_fwd(dy, wp, out=dx, out_place=(H * W, 2 * W, 2, a * W + b), out_hw_override=(Ho, Wo))
            sel = (slice(None), slice(a, None, 2), slice(b, None, 2))
        torch.cuda.synchronize()
        _check(name, G.mark(dx[sel]), r[sel], A[sel])
        G.check(name)


# ---- weight gradient ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", cc.WGRAD_CASES, ids=cc.case_id)
def test_wgrad_instances(c):
    """OHWI into zeros (twice: equal bytes), then OIHW added to a pre-loaded gradient"""
    from omni3d_b200 import conv as K
    inst, buckets, single = cc.wgrad_plan(cc.fwd_desc(c))
    name = f"wgrad {cc.case_id(c)} {inst} ncols {sorted(buckets)} {'one split' if single else 'splits'}"
    g = _gen(6)
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


# ---- fully-connected layers ------------------------------------------------------------------------------------------
def _lin_x(c, g):
    """x: the segments of a (rows, K) matrix whose gap rows hold the NaN pattern -> (guarded x, the segments stacked)"""
    total = (c.nseg - 1) * c.stride + c.rows
    G = Guarded(total * c.K, torch.bfloat16)
    xall = G.view((total, c.K))
    segs = []
    for s in range(c.nseg):
        v = G.mark(xall[s * c.stride:s * c.stride + c.rows])
        v.copy_(_bf(_randn(g, c.rows, c.K)))
        segs.append(v)
    return G, xall, torch.cat(segs)


@pytest.mark.parametrize("variant", ("bias_relu", "fp32"))
@pytest.mark.parametrize("c", cc.LINEAR_CASES, ids=cc.lin_id)
def test_linear_fwd(c, variant):
    from omni3d_b200 import _lib
    name = f"linear fwd {cc.lin_id(c)} {variant} ({cc.fwd_instance(cc.linear_descs(c)[0])})"
    g = _gen(7)
    Gx, xall, xs = _lin_x(c, g)
    w = _bf(_randn(g, c.N, c.K, scale=1 / math.sqrt(c.K)))
    b = _randn(g, c.N, scale=0.5)
    fp32 = variant == "fp32"
    r = xs.double() @ w.double().T + b.double()
    A = xs.double().abs() @ w.double().abs().T + b.double().abs()
    if not fp32:
        r = r.clamp_min(0)
    G = Guarded(c.nseg * c.rows * c.N, torch.float32 if fp32 else torch.bfloat16)
    y = G.mark(G.view((c.nseg * c.rows, c.N)))
    _lib.check(_lib.lib().c3d_linear_fwd(_lib.ptr(xall), _lib.ptr(w), _lib.ptr(b), _lib.ptr(y), c.nseg, c.rows, c.stride,
                                         c.K, c.N, int(not fp32), int(fp32), _lib.stream()))
    torch.cuda.synchronize()
    _check(name, y, r, A, fp32)
    G.check(name)
    Gx.check(name + " x")


@pytest.mark.parametrize("accumulate", (False, True), ids=("plain", "accumulate"))
@pytest.mark.parametrize("c", cc.LINEAR_CASES, ids=cc.lin_id)
def test_linear_dgrad(c, accumulate):
    from omni3d_b200 import conv as K
    g = _gen(8)
    dd = cc.linear_descs(c)[1]
    dd.add_mode = 3 if accumulate else 0
    name = f"linear dgrad {cc.lin_id(c)} {'accumulate' if accumulate else 'plain'} ({cc.fwd_instance(dd)})"
    dy = _bf(_randn(g, c.nseg * c.rows, c.N))
    w = _bf(_randn(g, c.N, c.K, scale=1 / math.sqrt(c.N)))
    r = dy.double() @ w.double()
    A = dy.double().abs() @ w.double().abs()
    total = (c.nseg - 1) * c.stride + c.rows
    G = Guarded(total * c.K, torch.bfloat16)
    dxall = G.view((total, c.K))
    segs = [G.mark(dxall[s * c.stride:s * c.stride + c.rows]) for s in range(c.nseg)]
    if accumulate:
        prior = _bf(_randn(g, c.nseg * c.rows, c.K))
        for s, v in enumerate(segs):
            v.copy_(prior[s * c.rows:(s + 1) * c.rows])
        r, A = r + prior.double(), A + prior.double().abs()
    K.linear_dgrad(dy, w.T.contiguous(), blocks=(c.nseg, c.rows, c.stride), dx=dxall, accumulate=accumulate)
    torch.cuda.synchronize()
    _check(name, torch.cat(segs), r, A)
    G.check(name)


@pytest.mark.parametrize("c", cc.LINEAR_CASES, ids=cc.lin_id)
def test_linear_wgrad(c):
    from omni3d_b200 import conv as K
    C, PP = c.chw if c.chw else (c.K, 1)
    inst, buckets, single = cc.wgrad_plan(cc.linear_descs(c)[0], C, PP)
    name = f"linear wgrad {cc.lin_id(c)} ({inst}, ncols {sorted(buckets)})"
    g = _gen(9)
    Gx, xall, xs = _lin_x(c, g)
    dy = _bf(_randn(g, c.nseg * c.rows, c.N))
    r = dy.double().T @ xs.double()                          # (N, K) in x's (p, c) feature order
    A = dy.double().abs().T @ xs.double().abs()
    r, A = (t.view(c.N, PP, C).transpose(1, 2).reshape(c.N, c.K) for t in (r, A))   # the master's (c, p) order
    G = Guarded(c.N * c.K, torch.float32)
    dw = G.mark(G.view((c.N, c.K)))
    dw_in = _randn(g, c.N, c.K, scale=r.abs().max().item())
    dw.copy_(dw_in)
    K.linear_wgrad(xall, dy, dw=dw, chw=c.chw, blocks=(c.nseg, c.rows, c.stride))
    torch.cuda.synchronize()
    cc.check(name, dw, r + dw_in.double(), A + dw_in.double().abs(), 0.0, cc.GAMMA_WGRAD)
    G.check(name)
    Gx.check(name + " x")
