"""GPU tests of the ROIAlign backward gather (c3d_roi_align_bwd) against a float64 torch scatter of the same samples."""
import ctypes
import math

import pytest
import torch

from omni3d_b200 import _lib
from omni3d_b200 import kernels as Kx

P = 7


def _fma(a, b, c):
    """fp32 a * b + c rounded once"""
    c = c.double() if torch.is_tensor(c) else c
    return (a.double() * b.double() + c).float()


def _ref_bwd(shapes, strides, rois, dout):
    """float64 (gradient, sum of |contributions|) per level: detectron2 ROIAlignV2 backward (aligned, adaptive sampling).
    The sample coordinates are rounded to fp32 like the kernel's (a fused multiply-add is exact in float64 before the one
    rounding to fp32), so the taps land on the same pixels; weights and sums are float64."""
    dev = rois.device
    grads = [torch.zeros(s, dtype=torch.float64, device=dev) for s in shapes]
    mags = [torch.zeros(s, dtype=torch.float64, device=dev) for s in shapes]
    r = rois.float()
    N, L = shapes[0][0], len(shapes)
    ok = torch.isfinite(r[:, 2:]).all(1) & (r[:, 0] >= 0) & (r[:, 0] < N) & (r[:, 1] >= 0) & (r[:, 1] < L)
    pp = torch.arange(P, device=dev, dtype=torch.float32)
    for lvl, (_, H, W, C) in enumerate(shapes):
        sel = (ok & (r[:, 1].clamp(0, L - 1).long() == lvl)).nonzero().flatten()
        if sel.numel() == 0:
            continue
        rr = r[sel]
        sc = torch.tensor(1.0 / strides[lvl], dtype=torch.float32, device=dev)
        sw, sh = _fma(rr[:, 2], sc, -0.5), _fma(rr[:, 3], sc, -0.5)
        rw, rh = _fma(rr[:, 4], sc, -0.5) - sw, _fma(rr[:, 5], sc, -0.5) - sh
        bw, bh = rw / torch.full_like(rw, P), rh / torch.full_like(rh, P)      # a true division, not x * (1 / P)
        gw, gh = torch.ceil(bw).long(), torch.ceil(bh).long()
        flat_g, flat_m = grads[lvl].view(-1, C), mags[lvl].view(-1, C)
        pairs = torch.unique(torch.stack([gh, gw], 1), dim=0).tolist()
        for a, c in pairs:
            if a <= 0 or c <= 0:
                continue
            sub = ((gh == a) & (gw == c)).nonzero().flatten()
            for part in sub.split(max(1, (1 << 17) // (P * P * a * c * 4))):
                def axis(s, b, n, size):
                    i = torch.arange(n, device=dev, dtype=torch.float32)
                    d = (i + 0.5)[None, None, :] * b[:, None, None]
                    v = _fma(pp[None, :, None], b[:, None, None], s[:, None, None]) + d / torch.full_like(d, n)
                    valid = (v >= -1.0) & (v <= size)
                    v = v.clamp(min=0.0)
                    lo = v.floor().long()
                    top = lo >= size - 1
                    lo = torch.where(top, torch.full_like(lo, size - 1), lo)
                    v = torch.where(top, lo.float(), v)
                    hi = torch.where(top, lo, lo + 1)
                    frac = (v - lo.float()).double()
                    idx = torch.stack([lo, hi], -1)                                # (n, P, samples, 2)
                    wt = torch.stack([1.0 - frac, frac], -1) * valid[..., None]
                    return idx, wt
                yi, yw = axis(sh[part], bh[part], a, H)
                xi, xw = axis(sw[part], bw[part], c, W)
                n = part.numel()
                img = rr[part, 0].long()
                pix = (img[:, None, None, None, None, None, None] * H + yi[:, :, :, :, None, None, None]) * W \
                    + xi[:, None, None, None, :, :, :]                            # (n, ph, iy, jy, pw, ix, jx)
                w = yw[:, :, :, :, None, None, None] * xw[:, None, None, None, :, :, :]
                g = dout[sel[part]].double() / max(a * c, 1)                      # (n, ph, pw, C)
                contrib = w[..., None] * g[:, :, None, None, :, None, None, :]
                flat_g.index_add_(0, pix.reshape(-1), contrib.reshape(-1, C))
                flat_m.index_add_(0, pix.reshape(-1), contrib.abs().reshape(-1, C))
                del contrib
    return grads, mags


def _check(got, ref, mag):
    for k, (a, b, m) in enumerate(zip(got, ref, mag)):
        err = (a.double() - b).abs()
        bad = err > 1e-4 * m + 1e-12
        assert not bad.any(), (k, int(bad.sum()), float(err.max()))


def _levels_shapes(N, C, sizes):
    return [(N, s, s, C) for s in sizes]


def _bwd_into(shapes, strides, rois, dout, fill):
    """call the library with maps pre-filled with `fill`: every element must be written"""
    feats = [torch.empty(s, device="cuda", dtype=torch.bfloat16) for s in shapes]
    grads = [torch.full(s, fill, device="cuda", dtype=torch.float32) for s in shapes]
    lv = Kx._levels(feats, strides, grads)
    _lib.check(_lib.lib().c3d_roi_align_bwd(ctypes.byref(lv), _lib.ptr(rois), rois.shape[0], shapes[0][3], P, P,
                                            _lib.ptr(dout), _lib.stream()))
    return grads


def _random_rois(N, per_image, S, gen, min_side=8.0, max_side=200.0):
    """FPN-assigned boxes like the box head's sampled proposals: log-uniform sides, level floor(4 + log2(sqrt(area) / 224))
    clamped to p2..p5 (index 0..3)."""
    R = N * per_image
    side = torch.exp(torch.empty(R, 2).uniform_(math.log(min_side), math.log(max_side), generator=gen))
    ctr = torch.rand(R, 2, generator=gen) * S
    x1, y1 = ctr[:, 0] - side[:, 0] / 2, ctr[:, 1] - side[:, 1] / 2
    x2, y2 = x1 + side[:, 0], y1 + side[:, 1]
    lvl = torch.floor(4 + torch.log2(torch.sqrt(side[:, 0] * side[:, 1]) / 224 + 1e-8)).clamp(2, 5) - 2
    img = torch.arange(N).repeat_interleave(per_image).float()
    return torch.stack([img, lvl, x1, y1, x2, y2], 1).float().cuda()


@pytest.mark.gpu
def test_flagship_shape_vs_float64_and_repeatable():
    gen = torch.Generator().manual_seed(0)
    N, S, C = 32, 640, 256
    strides = [4, 8, 16, 32]
    shapes = _levels_shapes(N, C, [S // s for s in strides])
    rois = _random_rois(N, 512, S, gen)
    dout = torch.randn(rois.shape[0], P, P, C, generator=gen).to(torch.bfloat16).cuda()
    feats = [torch.empty(s, device="cuda", dtype=torch.bfloat16) for s in shapes]
    a = Kx.roi_align_bwd(feats, strides, rois, dout)
    b = _bwd_into(shapes, strides, rois, dout, float("nan"))
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    ref, mag = _ref_bwd(shapes, strides, rois, dout)
    _check(a, ref, mag)


def _edge_case(case, gen):
    N, C = 2, 64
    strides = [4, 8]
    S = 128
    shapes = _levels_shapes(N, C, [S // s for s in strides])
    if case == "outside":          # boxes that straddle the image border or lie beyond it
        rois = _random_rois(N, 200, S, gen, 8.0, 120.0)
        rois[:, 2:] = rois[:, 2:] * 1.6 - 0.3 * S
        rois[:, 1] = torch.randint(0, 2, (rois.shape[0],), generator=gen).float().cuda()
    elif case == "degenerate":     # zero-size, NaN / Inf, bad level or image: no gradient from these
        rois = _random_rois(N, 64, S, gen, 8.0, 60.0)
        rois[:, 1] = torch.randint(0, 2, (rois.shape[0],), generator=gen).float().cuda()
        rois[0:8, 4] = rois[0:8, 2]
        rois[8:16, 5] = rois[8:16, 3]
        rois[16:20, 3] = float("nan")
        rois[20:24, 4] = float("inf")
        rois[24:28, 1] = 2.0
        rois[28:32, 0] = -1.0
        rois[32:36, 0] = N
    elif case == "whole_level":    # boxes covering a whole level, and more
        base = torch.tensor([[0, 0, 0, 0, S, S], [1, 0, -10, -10, S + 10, S + 10], [0, 1, 0, 0, S, S],
                             [1, 1, 3.5, 0, S - 2.25, S], [0, 0, -S, -S, 2 * S, 2 * S]], dtype=torch.float32)
        rois = torch.cat([base, _random_rois(N, 16, S, gen, 8.0, 60.0).cpu()]).cuda()
        rois[-32:, 1] = torch.randint(0, 2, (32,), generator=gen).float().cuda()
    elif case == "crowded":        # more than 2048 RoIs of one image and level reach one 8-row band
        R = 2600
        x1 = torch.rand(R, generator=gen) * (S - 40)
        y1 = 34.0 + torch.rand(R, generator=gen) * 4.0           # rows 8..9 at stride 4, band 1
        w = 8.0 + torch.rand(R, generator=gen) * 30.0
        rois = torch.stack([torch.zeros(R), torch.zeros(R), x1, y1, x1 + w, y1 + 12.0 + torch.rand(R, generator=gen) * 8.0], 1)
        rois = torch.cat([rois, _random_rois(N, 40, S, gen, 8.0, 60.0).cpu()]).cuda()
        rois[R:, 1] = torch.randint(0, 2, (rois.shape[0] - R,), generator=gen).float().cuda()
    elif case == "c512":
        C = 512
        shapes = _levels_shapes(N, C, [S // s for s in strides])
        rois = _random_rois(N, 128, S, gen, 8.0, 100.0)
        rois[:, 1] = torch.randint(0, 2, (rois.shape[0],), generator=gen).float().cuda()
    return shapes, strides, rois.contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["outside", "degenerate", "whole_level", "crowded", "c512"])
def test_edge_cases_vs_float64(case):
    gen = torch.Generator().manual_seed(1)
    shapes, strides, rois = _edge_case(case, gen)
    C = shapes[0][3]
    dout = torch.randn(rois.shape[0], P, P, C, generator=gen).to(torch.bfloat16).cuda()
    got = _bwd_into(shapes, strides, rois, dout, float("nan"))
    again = _bwd_into(shapes, strides, rois, dout, 0.0)
    for x, y in zip(got, again):
        assert torch.equal(x, y)
    ref, mag = _ref_bwd(shapes, strides, rois, dout)
    _check(got, ref, mag)
    if case == "degenerate":       # the insane RoIs alone give an all-zero gradient
        bad = torch.cat([rois[0:8], rois[8:16], rois[16:36]])
        dbad = torch.cat([dout[0:8], dout[8:16], dout[16:36]])
        for g in _bwd_into(shapes, strides, bad.contiguous(), dbad.contiguous(), float("nan")):
            assert torch.count_nonzero(g) == 0


@pytest.mark.gpu
def test_no_rois_gives_zero_maps():
    shapes = _levels_shapes(2, 64, [32, 16])
    rois = torch.zeros(0, 6, device="cuda")
    dout = torch.zeros(0, P, P, 64, device="cuda", dtype=torch.bfloat16)
    for g in _bwd_into(shapes, [4, 8], rois, dout, float("nan")):
        assert torch.count_nonzero(g) == 0
