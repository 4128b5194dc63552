"""Case table of the convolution / linear dispatch tests, with a Python mirror of the kernel-selection rules of
omni3d_b200/csrc/conv_tc.cu, conv_halo.cuh and nnfunc._dgrad, and the per-element error bound the tests apply.

The mirror lets a CPU test assert that the cases reach every compiled kernel instance and every data-gradient route
(tests/test_conv_dispatch_cpu.py), and that the instance lists below match the sources; the GPU tests
(tests/test_conv_dispatch_gpu.py) run the same cases against float64 references."""
import math
from types import SimpleNamespace

import torch

NUM_SMS = 132                                  # kNumSMs of c3d_common.cuh (H100 SXM)

# compiled instances, in source order
GEMM_FWD = [(256, 64), (128, 64), (64, 64), (32, 64), (16, 64), (128, 32), (64, 32), (32, 32), (16, 32),
            (128, 16), (64, 16), (32, 16), (16, 16)]                               # C3D_CONV_CASE (BLOCK_N, BLOCK_K)
HALO_FWD = [(1, 7, 8), (1, 3, 16), (1, 3, 32), (2, 7, 8), (2, 3, 16), (2, 3, 32)]  # C3D_HALO_F (Cout / 16, KH, Cin)
HALO_FWD_GENERIC = [(1, 0, 0), (2, 0, 0)]                                            # conv_halo_fwd_kernel<CH, 0, 0>
HALO_WGRAD = [(7, 8, 16), (7, 8, 32), (3, 16, 16), (3, 16, 32), (3, 32, 16), (3, 32, 32)]  # C3D_HALO_W (KH, Cin, Cout)
WGRAD_WIDTHS = (64, 32, 16)                    # cw (x channels per box) and ca (dy channels per box)
WGRAD_NCOLS = (64, 128, 192, 256)              # wgrad_consume<NB> accumulator widths
DGRAD_ROUTES = ("stride1", "merged", "merged_rows", "separate", "zero_stuff2")

# ---- error bound ---------------------------------------------------------------------------------------------------
# |got - r| <= q*|r| + gamma*A per element, r the float64 result of the bf16 operands as stored and A the same operation
# on |operands| (plus |bias|, |addend|, |prior buffer|).  q covers the final round-to-nearest to bf16 (8 significant
# bits: at most 2^-8 relative), so a bf16 output may use nearly all of q*|r|; gamma covers the fp32 accumulation of the
# tensor-core products and of the epilogue additions, and is the term a wrong tap, tile or bias trips.
# Measured on an H100 SXM (700 W) over every case of test_conv_dispatch_gpu.py, the largest
# max((|got - r| - q*|r|) / A) was 7.7e-7 for the forward / data gradient (the K = 12544 linear layer) and 2.2e-7
# for the weight gradient; the constants below leave 4.9x and 8.7x of headroom.
Q_BF16 = 2.0 ** -8
# forward / data gradient: fp32 sums of up to 12544 exact bf16 products per output
GAMMA_FWD = 2.0 ** -18
# weight gradient: fp32 sums over N*Ho*Wo pixels (up to 12288 here) in per-CTA accumulators, then the ordered fp32
# reduction of the split partials
GAMMA_WGRAD = 2.0 ** -19


def bound(r, A, q, gamma):
    return q * r.abs() + gamma * A


def worst_ratio(got, r, bnd):
    """largest |got - r| / bound over all elements (inf where the bound is 0 but the error is not, or got is NaN)"""
    err = (got.double() - r).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bnd)
    ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, math.inf), ratio)
    return ratio.max().item() if ratio.numel() else 0.0


def check(name, got, r, A, q, gamma):
    """assert the per-element bound; returns (worst err / bound, smallest gamma that would pass)"""
    bnd = bound(r, A, q, gamma)
    worst = worst_ratio(got, r, bnd)
    err = (got.double() - r).abs()
    need = torch.where(A > 0, (err - q * r.abs()).clamp_min(0) / A, torch.where(err > 0, math.inf, 0.0))
    need = torch.where(torch.isnan(need), torch.full_like(need, math.inf), need)
    g = need.max().item() if need.numel() else 0.0
    print(f"{name}: worst err/bound {worst:.3g}, gamma needed {g:.3g}")
    if not worst <= 1.0:
        bad = torch.nonzero(torch.where(torch.isnan(err), torch.full_like(err, math.inf), err) > bnd)[:5].tolist()
        raise AssertionError(f"{name}: err/bound {worst:.3g} > 1 at {bad} (got {[got[tuple(i)].item() for i in bad]}, "
                             f"ref {[r[tuple(i)].item() for i in bad]})")
    return worst, g


# ---- mirror of the selection rules -----------------------------------------------------------------------------------
def desc(N, H, W, Cin, Cout, k, stride=1, pad=0, add_mode=0, out_hw=None, x_img_stride=0, y_split_c=0,
         y_pix_stride=0):
    out_h, out_w = out_hw if out_hw is not None else (0, 0)
    return SimpleNamespace(N=N, H=H, W=W, Cin=Cin, Cout=Cout, KH=k, KW=k, stride=stride, pad=pad, add_mode=add_mode,
                           out_h=out_h, out_w=out_w, x_img_stride=x_img_stride, y_split_c=y_split_c,
                           y_pix_stride=y_pix_stride)


def out_size(d):
    Ho = d.out_h if d.out_h > 0 else (d.H + 2 * d.pad - d.KH) // d.stride + 1
    Wo = d.out_w if d.out_w > 0 else (d.W + 2 * d.pad - d.KW) // d.stride + 1
    return Ho, Wo


def _same_stride1(d):
    return d.stride == 1 and d.KH == d.KW and d.KH % 2 == 1 and 2 * d.pad == d.KH - 1


def _dense_images(d):
    # the halo kernels' tensor maps always use dense H*W image strides
    return d.N == 1 or d.x_img_stride in (0, d.H * d.W)


def halo_fwd_eligible(d):
    if not _same_stride1(d) or d.out_h > 0 or d.out_w > 0 or d.add_mode != 0:
        return False
    if d.Cin not in (8, 16, 32) or d.Cout not in (16, 32):
        return False
    if (d.W < 128 and d.Cin != 8) or d.KH > 7:
        return False
    return _dense_images(d) and d.y_split_c == 0


def halo_wgrad_eligible(d):
    if not _same_stride1(d) or d.Cin not in (8, 16, 32) or d.Cout not in (16, 32):
        return False
    if d.y_pix_stride not in (0, d.Cout) or (d.W < 128 and d.Cin != 8):
        return False
    return _dense_images(d) and ((d.KH == 7 and d.Cin == 8) or (d.KH == 3 and d.Cin >= 16))


def _width(c):
    return 64 if c % 64 == 0 else 32 if c % 32 == 0 else 16


def fwd_instance(d):
    """("halo", Cout/16, KS, CIN) with KS = CIN = 0 for the generic instances, or ("gemm", BLOCK_N, BLOCK_K)"""
    if halo_fwd_eligible(d):
        key = (d.Cout // 16, d.KH, d.Cin)
        return ("halo",) + (key if key in HALO_FWD else (d.Cout // 16, 0, 0))
    BK = _width(d.Cin)
    BN = 128 if d.Cout % 128 == 0 else _width(d.Cout)
    if BK == 64 and not (d.KH == 1 and d.Cin <= 64) and d.Cout % 256 == 0:
        BN = 256
    return ("gemm", BN, BK)


def _pick_tile_k(Ho, Wo, stride):
    best, bth, btw = -1.0, 1, 16
    for tw in range(1, 129):
        if tw * stride > 256:
            break
        if tw > Wo and tw != 16:
            continue
        th = 1
        while th * tw <= 128:
            if (th * tw) % 16 == 0 and th * stride <= 256:
                tiles = -(-Ho // th) * -(-Wo // tw)
                eff = Ho * Wo / (tiles * th * tw) * (1.0 if th * tw >= 64 else 0.9)
                if eff > best + 1e-9 or (eff > best - 1e-9 and th * tw > bth * btw):
                    best, bth, btw = eff, th, tw
            th += 1
    return bth, btw


def wgrad_plan(d, lin_c=0, lin_pp=0):
    """-> (instance, ncols buckets of the column groups, True if the grid has a single pixel split).
    instance: ("halo", KH, Cin, Cout) or ("gemm", cw, ca)."""
    if not lin_c and halo_wgrad_eligible(d):
        chunks = d.N * -(-d.W // 128) * -(-d.H // min(d.H, 32))
        return ("halo", d.KH, d.Cin, d.Cout), set(), chunks == 1
    Ho, Wo = out_size(d)
    cin_e, taps = (lin_c, lin_pp) if lin_c else (d.Cin, d.KH * d.KW)
    cw, ca = _width(cin_e), _width(d.Cout)
    bpc, total = 256 // cw, taps * (cin_e // cw)
    groups = -(-total // bpc)
    buckets = set()
    for g in range(groups):
        ncols = min(bpc, total - g * bpc) * cw
        buckets.add(next(nb for nb in WGRAD_NCOLS if ncols <= nb))
    RH, RW = _pick_tile_k(Ho, Wo, d.stride)
    num_tiles = d.N * -(-Ho // RH) * -(-Wo // RW)
    base = groups * -(-d.Cout // 128)
    splits = -(-4 * NUM_SMS // base) if d.Cout * taps * cin_e <= 65536 else NUM_SMS // base
    splits = max(1, min(splits, num_tiles))
    per = -(-num_tiles // splits)
    return ("gemm", cw, ca), buckets, -(-num_tiles // per) == 1


def merge_phases(I, O):                        # nnfunc._merge_phases
    return O <= 256 and (2 * I) % 16 == 0 and O % 16 == 0


def dgrad_route(c, into_slice):
    """route of nnfunc._dgrad for a dgrad case; into_slice: dx is a channel slice of a wider buffer"""
    Ho, Wo = out_size(desc(c.N, c.H, c.W, c.Cin, c.Cout, c.k, c.s, c.p))
    if c.s == 2 and c.k == 3 and c.p == 1 and c.H == 2 * Ho and c.W == 2 * Wo:
        if merge_phases(c.Cin, c.Cout):
            return "merged_rows" if into_slice else "merged"
        return "separate"
    return "stride1" if c.s == 1 else "zero_stuff2"


def dgrad_desc(c):
    """descriptor of the stride-1 convolution that computes a stride-1 data gradient (conv of dy with the rotated weight)"""
    Ho, Wo = out_size(desc(c.N, c.H, c.W, c.Cin, c.Cout, c.k, c.s, c.p))
    return desc(c.N, Ho, Wo, c.Cout, c.Cin, c.k, 1, c.k - 1 - c.p)


def linear_descs(c):
    """(forward, data-gradient) descriptors c3d_linear_fwd / c3d_linear_dgrad build"""
    f = desc(c.nseg, 1, c.rows, c.K, c.N, 1, x_img_stride=c.stride)
    g = desc(c.nseg, 1, c.rows, c.N, c.K, 1)
    return f, g


# ---- the cases ---------------------------------------------------------------------------------------------------------
def _case(**kw):
    kw.setdefault("N", 2)
    kw.setdefault("s", 1)
    kw.setdefault("p", kw["k"] // 2)
    kw.setdefault("out_hw", None)
    return SimpleNamespace(**kw)


def case_id(c):
    s = f"n{c.N}_{c.H}x{c.W}_c{c.Cin}-{c.Cout}_k{c.k}s{c.s}p{c.p}"
    return s + (f"_out{c.out_hw[0]}x{c.out_hw[1]}" if c.out_hw else "")


def fwd_desc(c, add_mode=0):
    return desc(c.N, c.H, c.W, c.Cin, c.Cout, c.k, c.s, c.p, add_mode=add_mode, out_hw=c.out_hw)


# one shape per GEMM instance; every one runs every epilogue variant of GEMM_VARIANTS (even outputs for up2)
GEMM_CASES = [
    _case(Cin=64, Cout=256, k=3, H=10, W=14),        # (256, 64)
    _case(Cin=64, Cout=256, k=1, H=10, W=14),        # (128, 64): 1x1 over <= 64 channels keeps BLOCK_N 128
    _case(Cin=192, Cout=192, k=3, s=2, H=12, W=16),  # (64, 64)
    _case(Cin=64, Cout=96, k=3, H=10, W=12),         # (32, 64)
    _case(Cin=128, Cout=48, k=1, H=8, W=8),          # (16, 64)
    _case(Cin=96, Cout=128, k=3, H=10, W=14),        # (128, 32)
    _case(Cin=32, Cout=64, k=3, H=10, W=14),         # (64, 32)
    _case(Cin=96, Cout=32, k=3, H=10, W=14),         # (32, 32)
    _case(Cin=32, Cout=48, k=3, H=10, W=14),         # (16, 32)
    _case(Cin=48, Cout=128, k=3, H=10, W=14),        # (128, 16)
    _case(Cin=16, Cout=64, k=3, H=10, W=14),         # (64, 16)
    _case(Cin=80, Cout=32, k=3, H=10, W=14),         # (32, 16)
    _case(Cin=16, Cout=16, k=3, H=10, W=14),         # (16, 16): W < 128 keeps it off the halo kernel
]
GEMM_VARIANTS = ("bias_relu_stats", "fp32", "addend", "up2", "acc_dense", "acc_slice")

# every halo forward instance: stride 1, same padding, W >= 128 unless Cin = 8 (the NHWC8 stem input)
HALO_CASES = [
    _case(Cin=8, Cout=16, k=7, H=5, W=130),
    _case(Cin=16, Cout=16, k=3, H=6, W=140),
    _case(Cin=32, Cout=16, k=3, N=1, H=35, W=128),   # two row chunks
    _case(Cin=8, Cout=32, k=7, H=4, W=100),
    _case(Cin=16, Cout=32, k=3, H=3, W=257),         # three strips, the last one 1 pixel wide
    _case(Cin=32, Cout=32, k=3, H=5, W=131),
    _case(Cin=16, Cout=16, k=1, H=3, W=150),         # generic <1,0,0>, KH = 1
    _case(Cin=32, Cout=16, k=5, H=6, W=129),         # generic <1,0,0>, KH = 5
    _case(Cin=8, Cout=16, k=3, H=7, W=60),           # generic <1,0,0>, Cin = 8, W < 128
    _case(Cin=32, Cout=32, k=1, H=3, W=200),         # generic <2,0,0>, KH = 1
    _case(Cin=16, Cout=32, k=5, H=6, W=133),         # generic <2,0,0>, KH = 5
    _case(Cin=8, Cout=32, k=3, H=5, W=77),           # generic <2,0,0>, Cin = 8, W < 128
]
HALO_VARIANTS = ("bias_relu", "fp32", "stats", "slice")

# edges of the GEMM path (bias + ReLU + statistics, bf16)
EDGE_CASES = [
    _case(Cin=64, Cout=64, k=3, N=1, H=5, W=7),              # one partial tile
    _case(Cin=32, Cout=64, k=3, H=1, W=37),                  # 1 x W output
    _case(Cin=32, Cout=64, k=3, H=37, W=1),                  # H x 1 output
    _case(Cin=64, Cout=128, k=3, s=2, H=13, W=11),           # odd sizes at stride 2
    _case(Cin=128, Cout=64, k=1, s=2, p=0, H=11, W=9),       # 1x1 stride 2, odd
    _case(Cin=48, Cout=64, k=3, p=0, H=9, W=12),             # pad 0
    _case(Cin=48, Cout=64, k=3, p=2, H=9, W=12),             # pad 2 > KH/2
    _case(Cin=64, Cout=32, k=3, H=9, W=10, out_hw=(12, 13)),           # high-side padding
    _case(Cin=32, Cout=16, k=3, s=2, H=12, W=12, out_hw=(7, 8)),
    _case(Cin=16, Cout=16, k=3, H=20, W=140, out_hw=(20, 140)),        # out_h/out_w set: GEMM even at halo widths
    _case(Cin=16, Cout=272, k=3, H=64, W=64),                # 17 N tiles, tiles_m x n_tiles = 4x the grid
    _case(Cin=64, Cout=384, k=3, H=10, W=14),                # 3 N tiles of 128
    _case(Cin=32, Cout=32, k=3, N=7, H=9, W=9),              # N = 7
]

# data gradient of y = conv(x, w, s, p), each dense, into a dense buffer and into a channel slice (`into=`)
DGRAD_CASES = [
    _case(Cin=64, Cout=32, k=1, H=9, W=10),
    _case(Cin=48, Cout=64, k=3, H=10, W=14),
    _case(Cin=16, Cout=32, k=7, H=9, W=11),
    _case(Cin=16, Cout=32, k=3, H=4, W=130),                 # dense: the halo kernel (Cin 32 -> Cout 16)
    _case(Cin=32, Cout=64, k=3, s=2, H=12, W=16),            # merged 2x2 (Cout <= 256)
    _case(Cin=64, Cout=256, k=3, s=2, H=8, W=10),
    _case(Cin=32, Cout=272, k=3, s=2, H=8, W=12),            # exact-FLOP separate phases (Cout > 256)
    _case(Cin=16, Cout=512, k=3, s=2, H=6, W=8),
    _case(Cin=32, Cout=64, k=3, s=2, H=13, W=12),            # zero_stuff2: odd H
    _case(Cin=32, Cout=64, k=3, s=2, H=12, W=11),            # zero_stuff2: odd W
    _case(Cin=64, Cout=128, k=1, s=2, p=0, H=12, W=16),      # zero_stuff2: 1x1 / s2, even
    _case(Cin=64, Cout=128, k=1, s=2, p=0, H=11, W=13),      # zero_stuff2: 1x1 / s2, odd
]
DGRAD_VARIANTS = ("dense", "into_dense", "into_slice")

# weight gradient: every (cw, ca) pair, the four accumulator widths, the halo instances, splits
WGRAD_CASES = [
    _case(Cin=64, Cout=64, k=3, H=10, W=14),                 # cw 64, ca 64: ncols 256 + 64
    _case(Cin=128, Cout=96, k=1, H=10, W=14),                # cw 64, ca 32: 128
    _case(Cin=64, Cout=48, k=3, H=9, W=9),                   # cw 64, ca 16
    _case(Cin=96, Cout=128, k=1, H=10, W=14),                # cw 32, ca 64
    _case(Cin=160, Cout=32, k=1, H=10, W=14),                # cw 32, ca 32: 160 -> 192
    _case(Cin=32, Cout=16, k=3, H=10, W=14),                 # cw 32, ca 16 (W < 128: GEMM)
    _case(Cin=48, Cout=192, k=3, H=10, W=14),                # cw 16, ca 64, two co tiles
    _case(Cin=16, Cout=96, k=3, H=10, W=14),                 # cw 16, ca 32
    _case(Cin=80, Cout=16, k=1, H=10, W=14),                 # cw 16, ca 16
    _case(Cin=16, Cout=16, k=3, H=5, W=127),                 # W = 127: GEMM fallback of a halo shape
    _case(Cin=32, Cout=64, k=3, s=2, H=13, W=11),            # stride 2, odd sizes
    _case(Cin=64, Cout=32, k=3, N=1, H=8, W=8),              # one tile: a single split adds into dw itself
    _case(Cin=16, Cout=32, k=3, N=4, H=48, W=64),            # many splits, small weight
    _case(Cin=64, Cout=256, k=3, H=32, W=48),                # many splits, > 64K weights
    _case(Cin=8, Cout=16, k=7, N=1, H=5, W=100),             # halo (7, 8, 16), one CTA
    _case(Cin=8, Cout=32, k=7, H=9, W=70),                   # halo (7, 8, 32)
    _case(Cin=16, Cout=16, k=3, H=40, W=130),                # halo (3, 16, 16), two row chunks
    _case(Cin=16, Cout=32, k=3, H=6, W=256),                 # halo (3, 16, 32)
    _case(Cin=32, Cout=16, k=3, H=6, W=140),                 # halo (3, 32, 16)
    _case(Cin=32, Cout=32, k=3, N=3, H=70, W=129),           # halo (3, 32, 32), many CTAs
]


def _lin(K, N, nseg, rows, stride, chw=None):
    return SimpleNamespace(K=K, N=N, nseg=nseg, rows=rows, stride=stride, chw=chw)


def lin_id(c):
    return f"K{c.K}_N{c.N}_seg{c.nseg}x{c.rows}of{c.stride}" + (f"_chw{c.chw[0]}x{c.chw[1]}" if c.chw else "")


LINEAR_CASES = [
    _lin(16, 16, 3, 128, 150),              # K, N in {16, 32}, >= 128 rows, strided segments: thin-channel widths
    _lin(16, 32, 3, 300, 333),
    _lin(32, 16, 3, 128, 129),
    _lin(32, 32, 3, 300, 420),
    _lin(32, 32, 1, 300, 310),              # one segment: the halo kernel, stride irrelevant
    _lin(16, 48, 3, 128, 140),
    _lin(48, 64, 3, 100, 117),
    _lin(64, 48, 1, 1, 1),
    _lin(1024, 16, 3, 1, 5),
    _lin(16, 1024, 3, 100, 130),
    _lin(1024, 1024, 1, 128, 160),
    _lin(64, 32, 3, 300, 310, chw=(16, 4)),
    _lin(256 * 49, 32, 3, 100, 112, chw=(256, 49)),
]
