"""ctypes front-end of the wgmma implicit-GEMM convolution entry points (include/c3d.h).

Tensors are torch CUDA tensors used as raw device buffers: activations NHWC bf16 (N,H,W,C),
weights OHWI bf16 (Cout,KH,KW,Cin).  No torch types cross the ABI.
"""
import ctypes

import torch

from . import _lib
from ._lib import ConvDesc, ptr, stream


def out_hw(H, W, KH, KW, stride, pad):
    return (H + 2 * pad - KH) // stride + 1, (W + 2 * pad - KW) // stride + 1


def make_desc(x, w, stride=1, pad=0, relu=False, out_fp32=False, add_mode=0):
    N, H, W, Cin = x.shape
    Cout, KH, KW, Cin2 = w.shape
    assert Cin == Cin2, (x.shape, w.shape)
    return ConvDesc(N=N, H=H, W=W, Cin=Cin, Cout=Cout, KH=KH, KW=KW, stride=stride, pad=pad, relu=int(relu),
                    out_fp32=int(out_fp32), add_mode=add_mode)


def num_tiles(desc):
    L = _lib.lib()
    t, th, tw = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32()
    _lib.check(L.c3d_conv2d_tiles(ctypes.byref(desc), ctypes.byref(t), ctypes.byref(th), ctypes.byref(tw)))
    return t.value, th.value, tw.value


def conv2d_fwd(x, w, bias=None, stride=1, pad=0, relu=False, addend=None, up2=False, out_fp32=False,
               want_stats=False, out=None, out_place=None, out_hw_override=None, accumulate=False, split=None):
    """x (N,H,W,Cin) bf16, w (Cout,KH,KW,Cin) bf16 -> y (N,Ho,Wo,Cout) bf16|fp32 [, stats (tiles,2,Cout)].
    out: write into this buffer (dense, or a channel slice of a wider NHWC tensor); accumulate: out += conv (add_mode 3,
    fp32 add in the epilogue) instead of out = conv."""
    L = _lib.lib()
    assert x.is_cuda and x.dtype == torch.bfloat16 and x.is_contiguous()
    assert w.dtype == torch.bfloat16 and w.is_contiguous()
    add_mode = 0 if addend is None else (2 if up2 else 1)
    if accumulate:
        assert addend is None and out is not None and not out_fp32 and not want_stats
        add_mode = 3
    d = make_desc(x, w, stride, pad, relu, out_fp32, add_mode)
    Ho, Wo = out_hw(d.H, d.W, d.KH, d.KW, stride, pad)
    if out_hw_override is not None:
        Ho, Wo = out_hw_override
        d.out_h, d.out_w = Ho, Wo
    if out_place is not None:        # (img_stride, h_stride, w_stride, offset) in pixels of `out`
        d.y_img_stride, d.y_h_stride, d.y_w_stride, d.y_offset = out_place
    if split is not None:            # (first channel of the second half, its extra offset in elements): c3d.h y_split_*
        d.y_split_c, d.y_split_off = split
    if out is None:
        out = torch.empty((d.N, Ho, Wo, d.Cout), device=x.device, dtype=torch.float32 if out_fp32 else torch.bfloat16)
    elif not out.is_contiguous():                      # channel slice of a wider NHWC buffer
        from .kernels import pixel_stride
        ps = pixel_stride(out)
        assert ps is not None, "conv2d_fwd: out must be dense or a 16-byte aligned channel slice"
        d.y_pix_stride = ps
    elif out.dim() == 4 and out.shape[-1] != d.Cout:   # split placement: the conv's channels span several pixels of `out`
        assert split is not None
        d.y_pix_stride = out.shape[-1]
    stats = None
    if want_stats:
        t, _, _ = num_tiles(d)
        stats = torch.empty((t, 2, d.Cout), device=x.device, dtype=torch.float32)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous()
    if addend is not None:
        assert addend.dtype == torch.bfloat16 and addend.is_contiguous()
    _lib.check(L.c3d_conv2d_fwd(ctypes.byref(d), ptr(x), ptr(w), ptr(bias), ptr(addend), ptr(out), ptr(stats),
                                stream()))
    return (out, stats) if want_stats else out


def pack_desc(w, want_fwd=True, want_dgrad=True, phases=None):
    """c3d_pack_desc of the fp32 master w (Cout,Cin,KH,KW), stored OIHW or channels_last, and the new bf16 outputs it points
    at -> (desc, (fwd, dgrad, phase packs)).  fwd (Cout,KH,KW,Cin); dgrad (Cin,KH,KW,Cout) rotated by 180 degrees; phases
    of a 3x3 weight: "separate" -> {(a, b): (Cin, 1 + a, 1 + b, Cout)}, "merged" -> the same keys as the row blocks of
    packs["merged"], one zeroed (4*Cin, 2, 2, Cout) weight whose unused taps the pack never writes (include/c3d.h)."""
    Cout, Cin, KH, KW = w.shape
    ohwi = (not w.is_contiguous()) and w.permute(0, 2, 3, 1).is_contiguous()
    if not (ohwi or w.is_contiguous()):
        raise ValueError("conv weight storage is neither OIHW nor channels_last")
    new = lambda *shape: torch.empty(shape, device=w.device, dtype=torch.bfloat16)
    f = new(Cout, KH, KW, Cin) if want_fwd else None
    g = new(Cin, KH, KW, Cout) if want_dgrad else None
    ph = None
    if phases == "merged":
        mg = torch.zeros((4 * Cin, 2, 2, Cout), device=w.device, dtype=torch.bfloat16)
        ph = {"merged": mg, **{(a, b): mg[(2 * a + b) * Cin:(2 * a + b + 1) * Cin] for a in (0, 1) for b in (0, 1)}}
    elif phases == "separate":
        ph = {(a, b): new(Cin, 1 + a, 1 + b, Cout) for a in (0, 1) for b in (0, 1)}
    elif phases is not None:
        raise ValueError(f"phases must be None, 'separate' or 'merged', not {phases!r}")
    d = _lib.PackDesc(src=w.data_ptr(), fwd=ptr(f), dgrad=ptr(g), Cout=Cout, Cin=Cin, KH=KH, KW=KW, src_is_ohwi=int(ohwi),
                      merged_phases=int(phases == "merged"))
    if ph is not None:
        d.phase = (ctypes.c_void_p * 4)(*[ph[(a, b)].data_ptr() for a in (0, 1) for b in (0, 1)])
    return d, (f, g, ph)


def pack_conv_weight(w, want_fwd=True, want_dgrad=True, phases=None):
    """fp32 (Cout,Cin,KH,KW) -> (bf16 fwd, bf16 dgrad, stride-2 phase packs | None) of pack_desc, in ONE launch."""
    w = w.detach()
    if not (w.is_contiguous() or w.permute(0, 2, 3, 1).is_contiguous()):
        w = w.contiguous()
    d, packs = pack_desc(w, want_fwd, want_dgrad, phases)
    _lib.check(_lib.lib().c3d_pack_conv_weight(ctypes.byref(d), stream()))
    return packs


def conv2d_wgrad(x, dy, KH, KW, stride=1, pad=0, dw=None, oihw=False):
    """dW (Cout,KH,KW,Cin) [or (Cout,Cin,KH,KW) when oihw] fp32 (+)= wgrad(x (N,H,W,Cin) bf16, dy bf16)."""
    L = _lib.lib()
    N, H, W, Cin = x.shape
    Cout = dy.shape[3]
    assert x.dtype == torch.bfloat16 and dy.dtype == torch.bfloat16 and x.is_contiguous() and dy.is_contiguous()
    if dw is None:
        dw = torch.zeros((Cout, Cin, KH, KW) if oihw else (Cout, KH, KW, Cin), device=x.device, dtype=torch.float32)
    d = ConvDesc(N=N, H=H, W=W, Cin=Cin, Cout=Cout, KH=KH, KW=KW, stride=stride, pad=pad)
    _lib.check(L.c3d_conv2d_wgrad(ctypes.byref(d), ptr(x), ptr(dy), ptr(dw), int(oihw), stream()))
    return dw


# ---- fully-connected layers on the same kernels (c3d_linear_*) -------------------------------------------------------
def pack_linear_weight(w, chw=None):
    """fp32 master (N, K) -> bf16 (N, K') and bf16 (K', N).  chw = (C, PP): the master's input features are ordered
    (c, p) (nn.Linear over an NCHW-flattened RoI) and are re-ordered to (p, c) (NHWC-flattened RoI)."""
    L = _lib.lib()
    N, Kdim = w.shape
    w = w.detach().contiguous()
    C, PP = chw if chw is not None else (Kdim, 1)
    f = torch.empty((N, Kdim), device=w.device, dtype=torch.bfloat16)
    t = torch.empty((Kdim, N), device=w.device, dtype=torch.bfloat16)
    _lib.check(L.c3d_pack_linear_weight(ptr(w), N, Kdim, C, PP, ptr(f), ptr(t), stream()), launches=2)
    return f, t


def _row_blocks(m, blocks):
    """(nseg, seg_rows, seg_stride) of the c3d_linear_* row blocks inside the (rows, ..) matrix m; blocks None: all rows"""
    rows = m.shape[0]
    nseg, seg_rows, seg_stride = blocks if blocks is not None else (1, rows, rows)
    assert (nseg - 1) * seg_stride + seg_rows <= rows, (blocks, tuple(m.shape))
    return nseg, seg_rows, seg_stride


def linear_fwd(x, w, bias=None, relu=False, out_fp32=False, blocks=None):
    """x (rows, K) bf16, w (N, K) bf16, bias (N,) fp32 -> [relu](x w^T + bias) (rows, N) bf16 | fp32.
    blocks = (nseg, seg_rows, seg_stride): only rows [b*seg_stride, b*seg_stride + seg_rows) of x, b < nseg, read in
    place -> (nseg*seg_rows, N)."""
    L = _lib.lib()
    Kdim, N = x.shape[1], w.shape[0]
    nseg, seg_rows, seg_stride = _row_blocks(x, blocks)
    assert x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and x.is_contiguous() and w.is_contiguous()
    assert w.shape[1] == Kdim and (bias is None or (bias.dtype == torch.float32 and bias.is_contiguous()))
    y = torch.empty((nseg * seg_rows, N), device=x.device, dtype=torch.float32 if out_fp32 else torch.bfloat16)
    _lib.check(L.c3d_linear_fwd(ptr(x), ptr(w), ptr(bias), ptr(y), nseg, seg_rows, seg_stride, Kdim, N, int(relu),
                                int(out_fp32), stream()))
    return y


def linear_dgrad(dy, wt, blocks=None, dx=None, accumulate=False):
    """dy (rows, N) bf16, wt (K, N) bf16 (the transposed weight) -> dx (rows, K) bf16 = dy . W.  dx: write into this
    buffer instead, at rows [b*seg_stride, +seg_rows) of blocks = (nseg, seg_rows, seg_stride); accumulate: dx +=."""
    L = _lib.lib()
    N, Kdim = dy.shape[1], wt.shape[0]
    assert dy.dtype == torch.bfloat16 and wt.dtype == torch.bfloat16 and dy.is_contiguous() and wt.is_contiguous()
    if dx is None:
        dx = torch.empty((dy.shape[0], Kdim), device=dy.device, dtype=torch.bfloat16)
    nseg, seg_rows, seg_stride = _row_blocks(dx, blocks)
    assert dx.dtype == torch.bfloat16 and dx.is_contiguous() and dx.shape[1] == Kdim and dy.shape[0] == nseg * seg_rows
    _lib.check(L.c3d_linear_dgrad(ptr(dy), ptr(wt), ptr(dx), nseg, seg_rows, seg_stride, N, Kdim, int(accumulate),
                                  stream()))
    return dx


def linear_wgrad(x, dy, dw=None, chw=None, blocks=None):
    """dw (N, K) fp32 (+)= dy^T x over the rows of x that blocks selects (as in linear_fwd).  chw = (C, PP): x's features
    are the (p, c) re-ordering of the master's (c, p) ones (pack_linear_weight), and dw is addressed in the master's order."""
    L = _lib.lib()
    Kdim, N = x.shape[1], dy.shape[1]
    nseg, seg_rows, seg_stride = _row_blocks(x, blocks)
    assert x.dtype == torch.bfloat16 and dy.dtype == torch.bfloat16 and x.is_contiguous() and dy.is_contiguous()
    if dw is None:
        dw = torch.zeros((N, Kdim), device=x.device, dtype=torch.float32)
    C, PP = chw if chw is not None else (Kdim, 1)
    _lib.check(L.c3d_linear_wgrad(ptr(x), ptr(dy), ptr(dw), nseg, seg_rows, seg_stride, Kdim, N, C, PP, stream()))
    return dw
