"""GPU tests of the ROIAlign backward's summation order and output types: the kernel's fp32 maps equal, bit for bit, the
host walk of the same contributions in (RoI, ph, pw, iy, ix, tap) order (tests/csrc/roi_align_host_harness.cpp); its
bf16 maps are those values rounded once; repeated calls give the same bytes."""
import pytest
import torch

import roi_harness as rh
from omni3d_b200 import _lib
from omni3d_b200 import kernels as Kx


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return rh.build(tmp_path_factory.mktemp("roi_harness"))


def _inputs(case, seed):
    gen = torch.Generator().manual_seed(seed)
    shapes, strides, rois = rh.flagship(gen) if case == "flagship" else rh.edge_case(case, gen)
    dout = torch.randn(rois.shape[0], rh.P, rh.P, shapes[0][3], generator=gen).to(torch.bfloat16)
    return shapes, strides, rois.cuda(), dout.cuda()


def _kernel(shapes, strides, rois, dout, dtype):
    feats = [torch.empty(s, device="cuda", dtype=torch.bfloat16) for s in shapes]
    return Kx.roi_align_bwd(feats, strides, rois, dout, rh.P, dtype=dtype)


def _check_fp32_against_host(harness, case, seed):
    shapes, strides, rois, dout = _inputs(case, seed)
    got = _kernel(shapes, strides, rois, dout, torch.float32)
    want = rh.bwd(harness, shapes, strides, rois, dout)
    for k, (a, b) in enumerate(zip(got, want)):
        a = a.cpu()
        b = torch.from_numpy(b)
        diff = a.view(torch.int32) != b.view(torch.int32)
        assert not diff.any(), (case, k, int(diff.sum()), float((a.double() - b.double()).abs().max()))
    assert any(torch.count_nonzero(a) for a in got) or case == "degenerate"


def _check_bf16_is_rounded_fp32(case, seed):
    shapes, strides, rois, dout = _inputs(case, seed)
    f32 = _kernel(shapes, strides, rois, dout, torch.float32)
    b16 = _kernel(shapes, strides, rois, dout, torch.bfloat16)
    again = _kernel(shapes, strides, rois, dout, torch.bfloat16)
    f32_again = _kernel(shapes, strides, rois, dout, torch.float32)
    for a, b, c, d in zip(f32, b16, again, f32_again):
        assert b.dtype == torch.bfloat16 and b.shape == a.shape
        assert torch.equal(b.view(torch.int16), a.to(torch.bfloat16).view(torch.int16))
        assert torch.equal(b.view(torch.int16), c.view(torch.int16))
        assert torch.equal(a.view(torch.int32), d.view(torch.int32))


@pytest.mark.gpu
def test_flagship_fp32_maps_equal_the_host_chain(harness):
    _check_fp32_against_host(harness, "flagship", 0)


@pytest.mark.gpu
@pytest.mark.parametrize("case", rh.CASES)
def test_edge_cases_fp32_maps_equal_the_host_chain(harness, case):
    _check_fp32_against_host(harness, case, 1)


@pytest.mark.gpu
def test_flagship_shape_bf16_maps_are_the_rounded_fp32_maps():
    _check_bf16_is_rounded_fp32("flagship", 2)


@pytest.mark.gpu
@pytest.mark.parametrize("case", rh.CASES)
def test_edge_cases_bf16_maps_are_the_rounded_fp32_maps(case):
    _check_bf16_is_rounded_fp32(case, 3)


@pytest.mark.gpu
def test_roi_align_bwd_rejects_other_dtypes():
    feats = [torch.empty(1, 8, 8, 64, device="cuda", dtype=torch.bfloat16)]
    rois = torch.zeros(0, 6, device="cuda")
    dout = torch.zeros(0, rh.P, rh.P, 64, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        Kx.roi_align_bwd(feats, [4], rois, dout, rh.P, dtype=torch.float16)


@pytest.mark.gpu
def test_misaligned_dout_is_rejected():
    shapes = rh.level_shapes(1, 64, [16])
    rois = torch.tensor([[0, 0, 4.0, 4.0, 40.0, 40.0]], device="cuda")
    flat = torch.zeros(rh.P * rh.P * 64 + 1, device="cuda", dtype=torch.bfloat16)
    dout = flat[1:].view(1, rh.P, rh.P, 64)                        # 2 bytes past a 16-byte boundary
    with pytest.raises(_lib.C3DError, match="16-byte aligned"):
        _kernel(shapes, [4], rois, dout, torch.float32)
