"""The case table of test_conv_dispatch_gpu.py against the sources (every compiled instance is listed and reached by a
case) and the per-element bound checker against seeded defects, on the CPU."""
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

import conv_cases as cc

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "omni3d_b200", "csrc")


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _tuples(pattern, text):
    return [tuple(int(v) for v in m) for m in re.findall(pattern, text, re.M)]


def test_instance_lists_match_the_sources():
    tc, halo = _source("conv_tc.cu"), _source("conv_halo.cuh")
    assert _tuples(r"^\s*C3D_CONV_CASE\((\d+),\s*(\d+),\s*\d+,\s*\d+\)", tc) == cc.GEMM_FWD
    assert _tuples(r"^\s*C3D_HALO_F\((\d+),\s*(\d+),\s*(\d+)\)", halo) == cc.HALO_FWD
    assert _tuples(r"launch_halo_fwd_inst<(\d+),\s*(\d+),\s*(\d+)>\(", halo) == cc.HALO_FWD_GENERIC
    assert _tuples(r"^\s*C3D_HALO_W\((\d+),\s*(\d+),\s*(\d+)\)", halo) == cc.HALO_WGRAD


def _fwd_descs():
    """every convolution descriptor the GPU cases launch through c3d_conv2d_fwd, with the case it belongs to"""
    add = {"addend": 1, "up2": 2, "acc_dense": 3, "acc_slice": 3}
    for c in cc.GEMM_CASES:
        for v in cc.GEMM_VARIANTS:
            yield c, cc.fwd_desc(c, add.get(v, 0))
    for c in cc.HALO_CASES + cc.EDGE_CASES:
        yield c, cc.fwd_desc(c)
    for c in cc.DGRAD_CASES:
        if cc.dgrad_route(c, False) == "stride1":
            yield c, cc.dgrad_desc(c)
    for c in cc.LINEAR_CASES:
        f, g = cc.linear_descs(c)
        yield c, f
        yield c, g
        g.add_mode = 3
        yield c, g


def test_cases_reach_every_forward_instance():
    assert [cc.fwd_instance(cc.fwd_desc(c)) for c in cc.GEMM_CASES] == [("gemm",) + i for i in cc.GEMM_FWD]
    halo = {("halo",) + i for i in cc.HALO_FWD + cc.HALO_FWD_GENERIC}
    assert {cc.fwd_instance(cc.fwd_desc(c)) for c in cc.HALO_CASES} == halo
    generic = {(c.k, c.Cin) for c in cc.HALO_CASES if cc.fwd_instance(cc.fwd_desc(c))[2] == 0}
    assert {(1, 16), (1, 32), (5, 16), (5, 32), (3, 8)} <= generic
    assert any(c.Cin == 8 and c.k == 3 and c.W < 128 for c in cc.HALO_CASES)
    reached = {cc.fwd_instance(d) for _, d in _fwd_descs()}
    assert reached >= halo | {("gemm",) + i for i in cc.GEMM_FWD}


def test_edge_cases_present():
    outs = [(c, cc.out_size(cc.fwd_desc(c))) for c in cc.EDGE_CASES]
    assert any(c.N * ho * wo < 128 for c, (ho, wo) in outs)
    assert any(ho == 1 for _, (ho, _) in outs) and any(wo == 1 for _, (_, wo) in outs)
    assert any(c.s == 2 and c.H % 2 and c.W % 2 for c in cc.EDGE_CASES)
    assert {0, 2} <= {c.p for c in cc.EDGE_CASES if c.k == 3}
    natural = lambda c: cc.out_size(cc.desc(c.N, c.H, c.W, c.Cin, c.Cout, c.k, c.s, c.p))
    assert any(c.out_hw and c.out_hw[0] > natural(c)[0] and c.out_hw[1] > natural(c)[1] for c in cc.EDGE_CASES)
    assert {272, 384} <= {c.Cout for c in cc.EDGE_CASES}
    assert {1, 7} <= {c.N for c in cc.EDGE_CASES}
    # tiles x N tiles several times the persistent grid (2 CTAs per SM below BLOCK_N 256)
    big = [c for c in cc.EDGE_CASES if c.Cout == 272][0]
    ho, wo = cc.out_size(cc.fwd_desc(big))
    assert big.N * ho * wo // 128 * (272 // cc.fwd_instance(cc.fwd_desc(big))[1]) >= 3 * 2 * cc.NUM_SMS


def test_cases_reach_every_dgrad_route():
    routes = {cc.dgrad_route(c, v == "into_slice") for c in cc.DGRAD_CASES for v in cc.DGRAD_VARIANTS}
    assert routes == set(cc.DGRAD_ROUTES)
    s1 = {c.k for c in cc.DGRAD_CASES if cc.dgrad_route(c, False) == "stride1"}
    assert {1, 3, 7} <= s1
    assert {272, 512} <= {c.Cout for c in cc.DGRAD_CASES if cc.dgrad_route(c, False) == "separate"}
    zs = [c for c in cc.DGRAD_CASES if cc.dgrad_route(c, False) == "zero_stuff2"]
    assert any(c.k == 3 and c.H % 2 for c in zs) and any(c.k == 3 and c.W % 2 for c in zs)
    assert any(c.k == 1 and c.H % 2 == 0 for c in zs) and any(c.k == 1 and c.H % 2 for c in zs)


def test_cases_reach_every_wgrad_instance():
    plans = [cc.wgrad_plan(cc.fwd_desc(c)) for c in cc.WGRAD_CASES]
    gemm = [p for p in plans if p[0][0] == "gemm"]
    halo = [p for p in plans if p[0][0] == "halo"]
    assert {p[0][1:] for p in gemm} == {(cw, ca) for cw in cc.WGRAD_WIDTHS for ca in cc.WGRAD_WIDTHS}
    assert set().union(*(p[1] for p in gemm)) == set(cc.WGRAD_NCOLS)
    assert {p[0][1:] for p in halo} == set(cc.HALO_WGRAD)
    for kind in (gemm, halo):               # one pixel split (dw += in the kernel) and several (ordered reduction)
        assert {p[2] for p in kind} == {True, False}
    fallback = [c for c in cc.WGRAD_CASES if c.Cin == 16 and c.W == 127]
    assert fallback and cc.wgrad_plan(cc.fwd_desc(fallback[0]))[0][0] == "gemm"
    assert any(c.s == 2 and c.H % 2 and c.W % 2 for c in cc.WGRAD_CASES)


def test_linear_cases():
    cs = cc.LINEAR_CASES
    assert {c.K for c in cs} >= {16, 32, 48, 64, 1024} and {c.N for c in cs} >= {16, 32, 48, 64, 1024}
    assert {c.nseg for c in cs} == {1, 3} and {c.rows for c in cs} >= {1, 100, 128, 300}
    assert all(c.stride > c.rows for c in cs if c.nseg > 1)
    assert {c.chw for c in cs} >= {(16, 4), (256, 49)}
    # the thin widths with strided segments: dense-image halo descriptors, so they must take the GEMM kernels
    thin = [c for c in cs if c.K in (16, 32) and c.N in (16, 32) and c.rows >= 128]
    assert {c.nseg > 1 and c.stride > c.rows for c in thin} == {True, False}
    for c in thin:
        f = cc.linear_descs(c)[0]
        assert cc.fwd_instance(f)[0] == ("gemm" if c.nseg > 1 else "halo"), cc.lin_id(c)


# ---- the bound checker against seeded defects --------------------------------------------------------------------
def _conv_case(seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 32, 10, 12, generator=g, dtype=torch.float64).bfloat16().double()
    w = (torch.randn(48, 32, 3, 3, generator=g, dtype=torch.float64) / math.sqrt(288)).bfloat16().double()
    b = torch.randn(48, generator=g, dtype=torch.float64).float().double()
    r = F.conv2d(x, w, b, padding=1)
    A = F.conv2d(x.abs(), w.abs(), b.abs(), padding=1)
    return x, w, b, r, A


def _fwd_ok(got, r, A):
    return cc.worst_ratio(got, r, cc.bound(r, A, cc.Q_BF16, cc.GAMMA_FWD)) <= 1.0


def test_bound_accepts_bf16_rounding():
    _, _, _, r, A = _conv_case()
    assert _fwd_ok(r.bfloat16().double(), r, A)
    assert _fwd_ok(r.float().double(), r, A)
    x, dy = torch.randn(2, 16, 9, 9, dtype=torch.float64), torch.randn(2, 32, 9, 9, dtype=torch.float64)
    rw = torch.nn.grad.conv2d_weight(x, (32, 16, 3, 3), dy, 1, 1)
    Aw = torch.nn.grad.conv2d_weight(x.abs(), (32, 16, 3, 3), dy.abs(), 1, 1)
    assert cc.worst_ratio(rw.float().double(), rw, cc.bound(rw, Aw, 0.0, cc.GAMMA_WGRAD)) <= 1.0


def test_bound_rejects_missing_k_block_on_border():
    x, w, b, r, A = _conv_case()
    wm = torch.zeros_like(w)
    wm[:, 16:32, 1, 1] = w[:, 16:32, 1, 1]        # one 16-channel K block of the centre tap
    part = F.conv2d(x, wm, None, padding=1)
    border = torch.zeros_like(r, dtype=torch.bool)
    border[:, :, 0, :] = border[:, :, -1, :] = border[:, :, :, 0] = border[:, :, :, -1] = True
    got = torch.where(border, r - part, r).bfloat16().double()
    assert not _fwd_ok(got, r, A)


def test_bound_rejects_pixel_shift_inside_one_tile():
    _, _, _, r, A = _conv_case()
    got = r.clone()
    got[1, :, 3, 1:] = r[1, :, 3, :-1]             # one output row of one tile shifted by a pixel
    assert not _fwd_ok(got.bfloat16().double(), r, A)


def test_bound_rejects_missing_bias_group():
    _, _, b, r, A = _conv_case()
    got = r.clone()
    got[:, 16:32] -= b[16:32].view(1, 16, 1, 1)
    assert not _fwd_ok(got.bfloat16().double(), r, A)


def test_bound_rejects_scaled_wgrad_row():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 16, 9, 9, generator=g, dtype=torch.float64).bfloat16().double()
    dy = torch.randn(2, 32, 9, 9, generator=g, dtype=torch.float64).bfloat16().double()
    r = torch.nn.grad.conv2d_weight(x, (32, 16, 3, 3), dy, 1, 1)
    A = torch.nn.grad.conv2d_weight(x.abs(), (32, 16, 3, 3), dy.abs(), 1, 1)
    got = r.float().double()
    got[5] *= 1 + 2.0 ** -6
    assert cc.worst_ratio(got, r, cc.bound(r, A, 0.0, cc.GAMMA_WGRAD)) > 1.0


def test_check_reports_nan():
    r = torch.ones(4, dtype=torch.float64)
    got = r.clone()
    got[2] = float("nan")
    with pytest.raises(AssertionError):
        cc.check("nan", got, r, r, cc.Q_BF16, cc.GAMMA_FWD)
