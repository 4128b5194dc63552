"""CPU tests of the exact host reference of the ROIAlign backward (tests/csrc/roi_align_host_harness.cpp), which the GPU
tests compare the kernel's maps against bit for bit: here it is checked against a float64 walk of the same samples."""
import math

import numpy as np
import pytest
import torch

import roi_harness as rh


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return rh.build(tmp_path_factory.mktemp("roi_harness"))


def _f32(x):
    return float(np.float32(x))


def _fma32(a, b, c):
    """fp32 a * b + c rounded once (the product of two fp32 values is exact in float64)"""
    return _f32(np.float64(a) * np.float64(b) + np.float64(c))


def _ref64(shapes, strides, rois, dout):
    """float64 (gradient, sum of |contributions|) per level: aligned ROIAlign backward with adaptive sampling; sample
    coordinates rounded to fp32 as the product rounds them, weights and sums in float64"""
    grads = [np.zeros(s) for s in shapes]
    mags = [np.zeros(s) for s in shapes]
    N, L = shapes[0][0], len(shapes)
    d = dout.float().numpy().astype(np.float64)
    for r, roi in enumerate(rois.tolist()):
        b, lvl = roi[0], roi[1]
        if not (all(math.isfinite(v) for v in roi[2:]) and 0 <= b < N and 0 <= lvl < L):
            continue
        b, lvl = int(b), int(lvl)
        _, H, W, _ = shapes[lvl]
        sc = _f32(1.0 / strides[lvl])
        sw, sh = _fma32(roi[2], sc, -0.5), _fma32(roi[3], sc, -0.5)
        width, height = _f32(_fma32(roi[4], sc, -0.5) - sw), _f32(_fma32(roi[5], sc, -0.5) - sh)
        bw, bh = _f32(width / rh.P), _f32(height / rh.P)
        gw, gh = math.ceil(bw), math.ceil(bh)
        cnt = max(gh * gw, 1)

        def axis(s, p, bb, i, n, size):
            v = _f32(_fma32(p, bb, s) + _f32(_f32((i + 0.5) * bb) / n))
            if v < -1.0 or v > size:
                return None
            v = max(v, 0.0)
            lo = int(v)
            if lo >= size - 1:
                return [(size - 1, 1.0), (size - 1, 0.0)]
            return [(lo, 1.0 - (v - lo)), (lo + 1, v - lo)]

        for ph in range(rh.P):
            for pw in range(rh.P):
                g = d[r, ph, pw] / cnt
                for iy in range(gh):
                    ys = axis(sh, ph, bh, iy, gh, H)
                    for ix in range(gw):
                        xs = axis(sw, pw, bw, ix, gw, W)
                        if ys is None or xs is None:
                            continue
                        for y, wy in ys:
                            for x, wx in xs:
                                grads[lvl][b, y, x] += wy * wx * g
                                mags[lvl][b, y, x] += abs(wy * wx * g)
    return grads, mags


def _small(gen):
    shapes = rh.level_shapes(2, 8, [16, 8])
    rois = rh.random_rois(2, 12, 64, gen, 4.0, 80.0)
    rois[:, 1] = torch.randint(0, 2, (rois.shape[0],), generator=gen).float()
    rois[0, 2:] = torch.tensor([-20.0, -20.0, 90.0, 90.0])          # beyond the image on every side
    rois[1, 4] = rois[1, 2]                                           # zero width
    rois[2, 3] = float("nan")
    rois[3, 0] = 2.0                                                  # image out of range
    return shapes, [4, 8], rois


def test_harness_matches_float64_walk(harness):
    gen = torch.Generator().manual_seed(5)
    shapes, strides, rois = _small(gen)
    dout = torch.randn(rois.shape[0], rh.P, rh.P, shapes[0][3], generator=gen).to(torch.bfloat16)
    got = rh.bwd(harness, shapes, strides, rois, dout)
    ref, mag = _ref64(shapes, strides, rois, dout)
    for a, b, m in zip(got, ref, mag):
        assert a.dtype == np.float32
        assert np.all(np.abs(a.astype(np.float64) - b) <= 1e-5 * m + 1e-12)
    assert any(np.count_nonzero(a) for a in got)


def test_harness_gives_zero_maps_for_rois_without_gradient(harness):
    gen = torch.Generator().manual_seed(6)
    shapes, strides, rois = _small(gen)
    bad = rois[1:4].contiguous()
    dout = torch.randn(bad.shape[0], rh.P, rh.P, shapes[0][3], generator=gen).to(torch.bfloat16)
    for a in rh.bwd(harness, shapes, strides, bad, dout):
        assert np.count_nonzero(a) == 0
