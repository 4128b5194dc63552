"""Inputs and the exact host reference of the ROIAlign backward tests.

`build(dir)` compiles tests/csrc/roi_align_host_harness.cpp (the product's sample geometry walked serially in the
kernel's contribution order) and `bwd` runs it; `random_rois` and `edge_case` make the RoI sets the tests use, on the
CPU, from a torch.Generator."""
import ctypes
import math
import os
import subprocess

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 7
CASES = ["outside", "degenerate", "whole_level", "crowded", "c512"]


def build(out_dir):
    out = os.path.join(str(out_dir), "libroi_harness.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "csrc", "roi_align_host_harness.cpp")])
    return ctypes.CDLL(out)


def bwd(lib, shapes, strides, rois, dout):
    """exact fp32 maps (numpy, shaped like `shapes`) for rois (R, 6) and bf16 dout (R, P, P, C), any device"""
    rois = np.ascontiguousarray(rois.detach().float().cpu().numpy())
    d = np.ascontiguousarray(dout.detach().float().cpu().numpy())
    N, C, L = shapes[0][0], shapes[0][3], len(shapes)
    maps = [np.empty(s, np.float32) for s in shapes]
    fp = ctypes.POINTER(ctypes.c_float)
    H = (ctypes.c_int * L)(*[s[1] for s in shapes])
    W = (ctypes.c_int * L)(*[s[2] for s in shapes])
    sc = (ctypes.c_float * L)(*[np.float32(1.0 / s) for s in strides])
    grads = (fp * L)(*[m.ctypes.data_as(fp) for m in maps])
    lib.harness_roi_align_bwd(rois.ctypes.data_as(fp), ctypes.c_int(rois.shape[0]), d.ctypes.data_as(fp), ctypes.c_int(C),
                              ctypes.c_int(P), ctypes.c_int(P), ctypes.c_int(N), ctypes.c_int(L), H, W, sc, grads)
    return maps


def level_shapes(N, C, sizes):
    return [(N, s, s, C) for s in sizes]


def random_rois(N, per_image, S, gen, min_side=8.0, max_side=200.0):
    """FPN-assigned boxes like the box head's sampled proposals: log-uniform sides, level floor(4 + log2(sqrt(area) / 224))
    clamped to p2..p5 (index 0..3)."""
    R = N * per_image
    side = torch.exp(torch.empty(R, 2).uniform_(math.log(min_side), math.log(max_side), generator=gen))
    ctr = torch.rand(R, 2, generator=gen) * S
    x1, y1 = ctr[:, 0] - side[:, 0] / 2, ctr[:, 1] - side[:, 1] / 2
    x2, y2 = x1 + side[:, 0], y1 + side[:, 1]
    lvl = torch.floor(4 + torch.log2(torch.sqrt(side[:, 0] * side[:, 1]) / 224 + 1e-8)).clamp(2, 5) - 2
    img = torch.arange(N).repeat_interleave(per_image).float()
    return torch.stack([img, lvl, x1, y1, x2, y2], 1).float()


def flagship(gen):
    """32 images at 640 x 640, 512 RoIs each, p2..p5 with 256 channels: (shapes, strides, rois)"""
    strides = [4, 8, 16, 32]
    return level_shapes(32, 256, [640 // s for s in strides]), strides, random_rois(32, 512, 640, gen)


def edge_case(case, gen):
    """(shapes, strides, rois) of two images at 128 x 128 on two levels"""
    N, C, S = 2, 64, 128
    strides = [4, 8]
    if case == "outside":          # boxes that straddle the image border or lie beyond it
        rois = random_rois(N, 200, S, gen, 8.0, 120.0)
        rois[:, 2:] = rois[:, 2:] * 1.6 - 0.3 * S
        rois[:, 1] = torch.randint(0, 2, (rois.shape[0],), generator=gen).float()
    elif case == "degenerate":     # zero-size, NaN / Inf, bad level or image: no gradient from these
        rois = random_rois(N, 64, S, gen, 8.0, 60.0)
        rois[:, 1] = torch.randint(0, 2, (rois.shape[0],), generator=gen).float()
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
        rois = torch.cat([base, random_rois(N, 16, S, gen, 8.0, 60.0)])
        rois[-32:, 1] = torch.randint(0, 2, (32,), generator=gen).float()
    elif case == "crowded":        # 2600 RoIs of one image and level on rows 8..9 of p2
        R = 2600
        x1 = torch.rand(R, generator=gen) * (S - 40)
        y1 = 34.0 + torch.rand(R, generator=gen) * 4.0
        w = 8.0 + torch.rand(R, generator=gen) * 30.0
        rois = torch.stack([torch.zeros(R), torch.zeros(R), x1, y1, x1 + w, y1 + 12.0 + torch.rand(R, generator=gen) * 8.0], 1)
        rois = torch.cat([rois, random_rois(N, 40, S, gen, 8.0, 60.0)])
        rois[R:, 1] = torch.randint(0, 2, (rois.shape[0] - R,), generator=gen).float()
    elif case == "c512":
        C = 512
        rois = random_rois(N, 128, S, gen, 8.0, 100.0)
        rois[:, 1] = torch.randint(0, 2, (rois.shape[0],), generator=gen).float()
    else:
        raise ValueError(case)
    return level_shapes(N, C, [S // s for s in strides]), strides, rois.contiguous()
