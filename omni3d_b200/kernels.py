"""ctypes front-ends of the NHWC helper kernels in libc3d.so (BatchNorm, max-pool, preprocess, ROIAlign,
SGD).  torch tensors are used only as device buffers; pointers + sizes cross the C ABI (include/c3d.h)."""
import ctypes

import torch

from . import _lib
from ._lib import ptr, stream

vp, i32, f32 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_float


def _bn_scratch(C, device):
    """the column-sum scratch of c3d_bn_finalize / c3d_bn_bwd / c3d_bias_act_bwd, of the size the library asks for"""
    return torch.empty(_lib.lib().c3d_bn_scratch_bytes(C), device=device, dtype=torch.uint8)


def bn_finalize(stats, count, eps, momentum, running_mean, running_var):
    L = _lib.lib()
    rows, _, C = stats.shape
    mean = torch.empty(C, device=stats.device, dtype=torch.float32)
    rstd = torch.empty(C, device=stats.device, dtype=torch.float32)
    scratch = _bn_scratch(C, stats.device)
    _lib.check(L.c3d_bn_finalize(ptr(stats), rows, C, float(count), eps, momentum, ptr(running_mean), ptr(running_var),
                                 ptr(mean), ptr(rstd), ptr(scratch), stream()), launches=1)
    return mean, rstd


def bn_apply(y, mean, rstd, gamma, beta, residual=None, relu=True, out=None):
    L = _lib.lib()
    C = y.shape[-1]
    P = y.numel() // C
    if out is None:
        out = torch.empty_like(y)
    _lib.check(L.c3d_bn_apply(ptr(y), ptr(mean), ptr(rstd), ptr(gamma), ptr(beta), ptr(residual), int(relu), ptr(out), P, C,
                              stream()))
    return out


def pixel_stride(t):
    """t (N,H,W,C) that is either dense or a channel slice of a dense NHWC buffer (what autograd hands back for the
    inputs of a torch.cat over channels) -> its pixel stride in elements, or None if it needs a .contiguous() copy."""
    if t.dim() != 4 or t.stride(3) != 1:
        return None
    N, H, W, C = t.shape
    s = t.stride(2)
    if s < C or s % 8 or (t.storage_offset() * t.element_size()) % 16:
        return None
    if (H > 1 and t.stride(1) != W * s) or (N > 1 and t.stride(0) != H * W * s):
        return None
    return s


def bn_bwd(dout, out, y, mean, rstd, gamma, relu, dgamma, dbeta, want_dres, frozen=False, beta=None, dres_into=None):
    """-> dy (bf16, like y), dres (bf16 or None); dgamma/dbeta (fp32 [C]) are accumulated in place.  `dout` may be a
    channel slice of a wider NHWC gradient (read in place through its pixel stride).  dres_into: an existing gradient
    buffer of the residual tensor (possibly a channel slice): the masked dout is ADDED into it in place."""
    L = _lib.lib()
    ds = pixel_stride(dout)
    if ds is None:
        dout, ds = dout.contiguous(), 0
    C = y.shape[-1]
    P = y.numel() // C
    blocks = L.c3d_bn_bwd_blocks(P, C)
    partial = torch.empty((blocks, 2, C), device=y.device, dtype=torch.float32)
    coef = torch.empty((3, C), device=y.device, dtype=torch.float32)
    dy = torch.empty_like(y)
    flags, rs = int(relu), 0
    if dres_into is not None:
        rs = pixel_stride(dres_into)
        assert rs is not None and dres_into.dtype == torch.bfloat16
        dres, flags = dres_into, flags | 2
    else:
        dres = torch.empty_like(y) if want_dres else None
    scratch = _bn_scratch(C, y.device)
    _lib.check(L.c3d_bn_bwd(ptr(dout), ptr(out), ptr(y), ptr(mean), ptr(rstd), ptr(gamma), ptr(beta), flags, int(frozen), ptr(partial), ptr(coef),
                            ptr(dgamma), ptr(dbeta), ptr(dy), ptr(dres), P, C, ds, rs, ptr(scratch), stream()), launches=3)
    return dy, dres


def maxpool2_fwd(x):
    L = _lib.lib()
    N, H, W, C = x.shape
    y = torch.empty((N, H // 2, W // 2, C), device=x.device, dtype=x.dtype)
    _lib.check(L.c3d_maxpool2_fwd(ptr(x), ptr(y), N, H, W, C, stream()))
    return y


def maxpool2_bwd(x, dy, into=None):
    """into: an existing gradient buffer of x (possibly a channel slice) that the routed dy is ADDED to in place."""
    L = _lib.lib()
    N, H, W, C = x.shape
    ds = pixel_stride(dy)
    if ds is None:
        dy, ds = dy.contiguous(), 0
    if into is None:
        dx, xs = torch.empty_like(x), 0
    else:
        dx, xs = into, pixel_stride(into)
        assert xs is not None and into.dtype == torch.bfloat16
    _lib.check(L.c3d_maxpool2_bwd(ptr(x), ptr(dy), ptr(dx), N, H, W, C, ds, xs, int(into is not None), stream()))
    return dx


def maxpool3s2_fwd(x):
    L = _lib.lib()
    N, H, W, C = x.shape
    y = torch.empty((N, (H - 1) // 2 + 1, (W - 1) // 2 + 1, C), device=x.device, dtype=x.dtype)
    _lib.check(L.c3d_maxpool3s2_fwd(ptr(x), ptr(y), N, H, W, C, stream()))
    return y


def maxpool3s2_bwd(x, dy):
    L = _lib.lib()
    N, H, W, C = x.shape
    ds = pixel_stride(dy)
    if ds is None:
        dy, ds = dy.contiguous(), 0
    dx = torch.empty_like(x)
    _lib.check(L.c3d_maxpool3s2_bwd(ptr(x), ptr(dy), ptr(dx), N, H, W, C, ds, stream()))
    return dx


def preprocess_images(images, mean, std, size_divisibility=64, cpad=16):
    """list of (3,H,W) fp32 or uint8 CUDA tensors -> (N,Hp,Wp,cpad) bf16 NHWC batch (normalised, zero padded)."""
    L = _lib.lib()
    Hm = max(im.shape[1] for im in images)
    Wm = max(im.shape[2] for im in images)
    d = size_divisibility
    Hp, Wp = (Hm + d - 1) // d * d, (Wm + d - 1) // d * d
    out = torch.empty((len(images), Hp, Wp, cpad), device=images[0].device, dtype=torch.bfloat16)
    m = (f32 * 3)(*[float(v) for v in mean])
    s = (f32 * 3)(*[float(v) for v in std])
    for im in images:
        assert im.dtype in (torch.float32, torch.uint8) and im.is_contiguous() and im.is_cuda

    def run(ims, dst):
        n = len(ims)
        ptrs = (vp * n)(*[im.data_ptr() for im in ims])
        hs = (i32 * n)(*[im.shape[1] for im in ims])
        ws = (i32 * n)(*[im.shape[2] for im in ims])
        _lib.check(L.c3d_preprocess_batch(ptrs, hs, ws, n, int(ims[0].dtype == torch.uint8), ptr(dst), Hp, Wp, cpad, m, s,
                                          stream()), launches=(n + 63) // 64)
    if all(im.dtype == images[0].dtype for im in images):     # the usual case: one launch for the whole batch
        run(images, out)
    else:                                                    # uint8 and fp32 images mixed: one launch per image
        for i, im in enumerate(images):
            run([im], out[i])
    return out


def _levels(feats, strides, grads=None):
    lv = _lib.RoiLevels()
    lv.num_levels = len(feats)
    lv.num_images = feats[0].shape[0]
    for i, f in enumerate(feats):
        lv.feat[i] = f.data_ptr()
        lv.grad[i] = grads[i].data_ptr() if grads is not None else None
        lv.H[i], lv.W[i] = f.shape[1], f.shape[2]
        lv.scale[i] = 1.0 / strides[i]
    return lv


def roi_align_fwd(feats, strides, rois, pooled=7):
    """feats: list of (N,H,W,C) bf16; rois (R,6) fp32 [batch, level, x1,y1,x2,y2] -> (R,pooled,pooled,C) bf16."""
    L = _lib.lib()
    C = feats[0].shape[-1]
    R = rois.shape[0]
    out = torch.empty((R, pooled, pooled, C), device=feats[0].device, dtype=torch.bfloat16)
    lv = _levels(feats, strides)
    _lib.check(L.c3d_roi_align_fwd(ctypes.byref(lv), ptr(rois), R, C, pooled, pooled, ptr(out), stream()))
    return out


def roi_align_bwd(feats, strides, rois, dout, pooled=7):
    """-> list of fp32 gradient maps shaped like feats (the kernel writes every element)."""
    L = _lib.lib()
    C = feats[0].shape[-1]
    grads = [torch.empty(f.shape, device=f.device, dtype=torch.float32) for f in feats]
    lv = _levels(feats, strides, grads)
    _lib.check(L.c3d_roi_align_bwd(ctypes.byref(lv), ptr(rois), rois.shape[0], C, pooled, pooled, ptr(dout), stream()))
    return grads


def grad_finite(flat_grad, flag):
    L = _lib.lib()
    _lib.check(L.c3d_grad_finite(ptr(flat_grad), flat_grad.numel(), ptr(flag), stream()))


def sgd_momentum(p, g, mom, lr, momentum, weight_decay, grad_scale=1.0, skip_flag=None):
    """lr: python float, or a 1-element fp32 CUDA tensor (read by the kernel at run time: CUDA-graph friendly)."""
    L = _lib.lib()
    lr_dev, lr = (lr, 0.0) if torch.is_tensor(lr) else (None, lr)
    _lib.check(L.c3d_sgd_momentum(ptr(p), ptr(g), ptr(mom), p.numel(), lr, ptr(lr_dev), momentum, weight_decay, grad_scale,
                                  ptr(skip_flag), stream()))


_nms_ws = {}


def nms_batched(boxes, nvalid, iou_thresh, max_keep, cats=None, maxc=None, trick_max_numel=20000, ncat=0, max_per_cat=0):
    """boxes (B,n,4) fp32 sorted by score desc, nvalid (B,) int32, cats (B,n) fp32 categories, maxc (B,) fp32
    -> keep_idx (B,max_keep) int32 (-1 padded, score order), keep_cnt (B,) int32.  No host sync.
    ncat > 0: the categories are exactly the integers 0..ncat-1 -> per-category kernels (same result, less work)."""
    L = _lib.lib()
    B, n, _ = boxes.shape
    boxes = boxes.contiguous()
    need = L.c3d_nms_workspace_bytes(B, n)
    key = boxes.device.index
    ws = _nms_ws.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.uint8, device=boxes.device)
        _nms_ws[key] = ws
    keep = torch.empty((B, max_keep), dtype=torch.int32, device=boxes.device)
    cnt = torch.empty((B,), dtype=torch.int32, device=boxes.device)
    if ncat > 0 and cats is not None:
        _lib.check(L.c3d_nms_batched_grouped(ptr(boxes), ptr(nvalid), ptr(cats), ptr(maxc), trick_max_numel, B, n, iou_thresh,
                                             max_keep, ncat, max_per_cat, ptr(keep), ptr(cnt), ptr(ws), ws.numel(), stream()),
                   launches=4)
        return keep, cnt
    _lib.check(L.c3d_nms_batched(ptr(boxes), ptr(nvalid), ptr(cats), ptr(maxc), trick_max_numel, B, n, iou_thresh,
                                 max_keep, ptr(keep), ptr(cnt), ptr(ws), ws.numel(), stream()), launches=2)
    return keep, cnt


def anchor_match(anchors, gt_boxes, gt_valid, gt_ign, fg_thresh):
    """anchors (A,4), gt_boxes (B,G,4) fp32, gt_valid / gt_ign (B,G) bool -> matched_idx (B,A) int64, matched_iou (B,A),
    labels (B,A) int8 {0,1}, max_ioa (B,A), best_idx (B,G) int32 (A for non-valid GTs)."""
    L = _lib.lib()
    A = anchors.shape[0]
    B, G, _ = gt_boxes.shape
    dev = anchors.device
    anchors, gt_boxes = anchors.contiguous().float(), gt_boxes.contiguous().float()
    v8, i8 = gt_valid.to(torch.uint8).contiguous(), gt_ign.to(torch.uint8).contiguous()
    idx = torch.empty((B, A), dtype=torch.int64, device=dev)
    iou = torch.empty((B, A), dtype=torch.float32, device=dev)
    ioa = torch.empty((B, A), dtype=torch.float32, device=dev)
    lab = torch.empty((B, A), dtype=torch.int8, device=dev)
    best = torch.empty((B, G), dtype=torch.int32, device=dev)
    ws = torch.empty((B, G), dtype=torch.int32, device=dev)
    _lib.check(L.c3d_anchor_match(ptr(anchors), A, ptr(gt_boxes), ptr(v8), ptr(i8), B, G, float(fg_thresh), ptr(idx), ptr(iou),
                                  ptr(lab), ptr(ioa), ptr(best), ptr(ws), stream()), launches=3)
    return idx, iou, lab, ioa, best


def rpn_decode_level(topk_idx, topk_score, deltas, anchors, image_hw, weights, scale_clamp, min_size, level, col0, boxes,
                     key, lvl, nvalid, maxc):
    """decode one level's top-k candidates into columns col0.. of boxes (B,Ktot,4) / key / lvl (B,Ktot); nvalid (B,) int32
    and maxc (B,) fp32 accumulate (zero them first)."""
    L = _lib.lib()
    B, K = topk_idx.shape
    w = (f32 * 4)(*[float(v) for v in weights])
    assert topk_idx.dtype == torch.int64 and topk_idx.stride(1) == 1 and topk_score.stride() == topk_idx.stride()
    _lib.check(L.c3d_rpn_decode_level(ptr(topk_idx), ptr(topk_score), topk_idx.stride(0), ptr(deltas), ptr(anchors), ptr(image_hw), B, K,
                                      deltas.shape[1], w, float(scale_clamp), float(min_size), int(level), int(col0),
                                      boxes.shape[1], ptr(boxes), ptr(key), ptr(lvl), ptr(nvalid), ptr(maxc), stream()))


def rpn_loss_fwd(logits, deltas, labels, matched_idx, gt_boxes, anchors, weights):
    """-> acc (6,) fp32: [sum cls, sum loc, #pos, #neg, sum sigmoid over positives, sum sigmoid over the rest]."""
    L = _lib.lib()
    B, A = logits.shape
    acc = torch.empty(6, dtype=torch.float32, device=logits.device)
    w = (f32 * 4)(*[float(v) for v in weights])
    _lib.check(L.c3d_rpn_loss_fwd(ptr(logits), ptr(deltas), ptr(labels), ptr(matched_idx), ptr(gt_boxes), ptr(anchors), B, A,
                                  gt_boxes.shape[1], w, ptr(acc), stream()))
    return acc


def rpn_loss_bwd(logits, deltas, labels, matched_idx, gt_boxes, anchors, weights, g_cls, g_loc):
    L = _lib.lib()
    B, A = logits.shape
    dl = torch.empty_like(logits)
    dd = torch.empty_like(deltas)
    w = (f32 * 4)(*[float(v) for v in weights])
    _lib.check(L.c3d_rpn_loss_bwd(ptr(logits), ptr(deltas), ptr(labels), ptr(matched_idx), ptr(gt_boxes), ptr(anchors), B, A,
                                  gt_boxes.shape[1], w, ptr(g_cls), ptr(g_loc), ptr(dl), ptr(dd), stream()))
    return dl, dd


def bias_act_bwd(dout, out, relu, dbias):
    """dz (bf16) = dout * (out > 0 if relu); dbias (fp32 [C] or None) += sum over pixels."""
    L = _lib.lib()
    C = dout.shape[-1]
    P = dout.numel() // C
    dout = dout.contiguous()
    blocks = L.c3d_bn_bwd_blocks(P, C)
    partial = torch.empty((blocks, C), device=dout.device, dtype=torch.float32)
    scratch = _bn_scratch(C, dout.device)
    alias = (not relu) and dout.dtype == torch.bfloat16          # no activation: dz IS dout, only the bias gradient is left
    if alias and dbias is None:
        return dout
    dz = None if alias else torch.empty(dout.shape, device=dout.device, dtype=torch.bfloat16)
    flags = int(dout.dtype == torch.float32) | (2 if (out is not None and out.dtype == torch.float32) else 0)
    _lib.check(L.c3d_bias_act_bwd(ptr(dout), ptr(out), int(relu), flags, ptr(dz), ptr(partial),
                                  ptr(dbias), P, C, ptr(scratch), stream()), launches=2 if dbias is not None else 1)
    return dout if alias else dz


def sumpool2(x):
    L = _lib.lib()
    N, H, W, C = x.shape
    y = torch.empty((N, H // 2, W // 2, C), device=x.device, dtype=x.dtype)
    _lib.check(L.c3d_sumpool2(ptr(x), ptr(y), N, H, W, C, stream()))
    return y


def zero_stuff2(dy, H, W):
    L = _lib.lib()
    N, Ho, Wo, C = dy.shape
    z = torch.empty((N, H, W, C), device=dy.device, dtype=dy.dtype)
    _lib.check(L.c3d_zero_stuff2(ptr(dy), ptr(z), N, Ho, Wo, H, W, C, stream()))
    return z


def cube_loss_fwd(raw, aux):
    L = _lib.lib()
    n = raw.shape[0]
    out = torch.empty((n, 10), device=raw.device, dtype=torch.float32)
    _lib.check(L.c3d_cube_loss_fwd(ptr(raw), ptr(aux), n, ptr(out), stream()))
    return out


def cube_loss_bwd(raw, aux, dout):
    L = _lib.lib()
    n = raw.shape[0]
    draw = torch.empty((n, 13), device=raw.device, dtype=torch.float32)
    _lib.check(L.c3d_cube_loss_bwd(ptr(raw), ptr(aux), ptr(dout), n, ptr(draw), stream()))
    return draw


# ---- selection / sampling (select_ops.cu) ----------------------------------------------------------------------------
_rng_state = {}


def rng_state(device, seed=None):
    """{seed, step counter} (2 x int64) on the device: the Philox stream of the sampling kernels.  The counter is advanced
    BY the kernels, so a CUDA-graph replay draws fresh noise every step without any host write."""
    key = (device.type, device.index)
    st = _rng_state.get(key)
    if st is None or seed is not None:
        if seed is None:
            seed = torch.initial_seed()
            try:
                import torch.distributed as dist
                if dist.is_available() and dist.is_initialized():
                    seed += 7919 * dist.get_rank()
            except Exception:      # noqa: BLE001
                pass
        st = _rng_state[key] = torch.tensor([seed & 0x7fffffffffffffff, 0], dtype=torch.int64, device=device)
    return st


def topk_segments(segs, want_idx64=False, want_counts=False):
    """segs: list of (vals (B,n) fp32 [row-strided ok], k).  -> vals (B, sum k) sorted descending inside every segment,
    idx (B, sum k) int32 or int64 (index inside the segment's row) [, counts (B, nseg) of values > -inf]."""
    L = _lib.lib()
    B = segs[0][0].shape[0]
    dev = segs[0][0].device
    arr = (_lib.TopkSeg * len(segs))()
    col = 0
    keep = []
    for i, (v, k) in enumerate(segs):
        assert v.dtype == torch.float32 and v.dim() == 2 and v.stride(1) == 1 and v.shape[0] == B
        keep.append(v)
        arr[i].vals, arr[i].row_stride, arr[i].n, arr[i].k, arr[i].out_col = v.data_ptr(), v.stride(0), v.shape[1], int(k), col
        col += int(k)
    out_v = torch.empty((B, col), dtype=torch.float32, device=dev)
    out_i = torch.empty((B, col), dtype=torch.int64 if want_idx64 else torch.int32, device=dev)
    cnt = torch.empty((B, len(segs)), dtype=torch.int32, device=dev) if want_counts else None
    _lib.check(L.c3d_topk_segments(arr, len(segs), B, col, ptr(out_v), None if want_idx64 else ptr(out_i),
                                   ptr(out_i) if want_idx64 else None, ptr(cnt), stream()))
    return (out_v, out_i, cnt) if want_counts else (out_v, out_i)


def label_sample_proposals(prop_boxes, prop_count, gt, K, S, Fcap, iou_thresh, ignore_thresh, append_gt=True, rng=None,
                           bump_rng=True, want_prelabels=False, want_index=False):
    """-> dict(boxes (B,S,4), valid (B,S) bool, classes (B,S) int64, gt_boxes, gt_boxes3D (B,S,9), gt_poses (B,S,3,3),
    stats (2,) [, index (B,S)] [, pre = (matched_idx, matched_iou, labels) each (B,P+G)])."""
    L = _lib.lib()
    B, P, _ = prop_boxes.shape
    G = gt["boxes"].shape[1]
    dev = prop_boxes.device
    f = lambda t: t.contiguous().float()
    pb, gb, g3, gp = f(prop_boxes), f(gt["boxes"]), f(gt["boxes3D"][..., :9]), f(gt["poses"].reshape(B, G, 9))
    pc = prop_count.to(torch.int32).contiguous()
    gc = gt["classes"].to(torch.int64).contiguous()
    pres = gt["present"].to(torch.uint8).contiguous()
    n = P + (G if append_gt else 0)
    out = dict(boxes=torch.empty((B, S, 4), device=dev), valid=torch.empty((B, S), dtype=torch.uint8, device=dev),
               classes=torch.empty((B, S), dtype=torch.int64, device=dev), gt_boxes=torch.empty((B, S, 4), device=dev),
               gt_boxes3D=torch.empty((B, S, 9), device=dev), gt_poses=torch.empty((B, S, 3, 3), device=dev),
               stats=torch.zeros(2, device=dev))
    pre = None
    if want_prelabels:
        pre = (torch.empty((B, n), dtype=torch.int64, device=dev), torch.empty((B, n), device=dev),
               torch.empty((B, n), dtype=torch.int64, device=dev))
    idx = torch.empty((B, S), dtype=torch.int64, device=dev) if want_index else None
    if rng is None:
        rng = rng_state(dev)
    a = _lib.LabelSampleArgs()
    a.prop_boxes, a.prop_count, a.gt_boxes, a.gt_classes, a.gt_present = pb.data_ptr(), pc.data_ptr(), gb.data_ptr(), gc.data_ptr(), pres.data_ptr()
    a.gt_boxes3D, a.gt_poses = g3.data_ptr(), gp.data_ptr()
    a.B, a.P, a.G, a.K, a.S, a.Fcap, a.append_gt = B, P, G, int(K), int(S), int(Fcap), int(bool(append_gt))
    a.iou_thresh, a.ignore_thresh = float(iou_thresh), float(ignore_thresh)
    a.rng, a.bump_rng = rng.data_ptr(), int(bool(bump_rng))
    if pre is not None:
        a.matched_idx, a.matched_iou, a.labels = pre[0].data_ptr(), pre[1].data_ptr(), pre[2].data_ptr()
    a.s_boxes, a.s_valid, a.s_classes = out["boxes"].data_ptr(), out["valid"].data_ptr(), out["classes"].data_ptr()
    a.s_gt_boxes, a.s_gt_boxes3D, a.s_gt_poses = out["gt_boxes"].data_ptr(), out["gt_boxes3D"].data_ptr(), out["gt_poses"].data_ptr()
    a.s_index = idx.data_ptr() if idx is not None else None
    a.stats = out["stats"].data_ptr()
    _lib.check(L.c3d_label_sample_proposals(ctypes.byref(a), stream()), launches=2 if bump_rng else 1)
    out["valid"] = out["valid"].view(torch.bool)
    if idx is not None:
        out["index"] = idx
    if pre is not None:
        out["pre"] = pre
    return out


def anchor_sample(labels01, matched_iou, max_ioa, best_idx, gt_valid, gt_ign, n_total, cap_pos, ignore_thresh, rng=None,
                  bump_rng=True):
    """labels01 (B,A) int8 matcher labels {0,1} -> sampled labels (B,A) int8 in {-1,0,1} (rpn.py:62-105)."""
    L = _lib.lib()
    B, A = labels01.shape
    dev = labels01.device
    G = gt_valid.shape[1]
    if rng is None:
        rng = rng_state(dev)
    keys = torch.empty((B, 2, A), dtype=torch.float32, device=dev)
    counts = torch.empty((B, 2), dtype=torch.int32, device=dev)
    lab = labels01.contiguous()
    _lib.check(L.c3d_anchor_sample_keys(ptr(lab), ptr(matched_iou.contiguous()), B, A, ptr(rng), ptr(keys), ptr(counts), stream()))
    k = int(max(cap_pos, n_total))
    kv = keys.view(B, 2 * A)
    _, idx = topk_segments([(kv[:, :A], k), (kv[:, A:], k)])
    out = torch.empty((B, A), dtype=torch.int8, device=dev)
    v8, i8 = gt_valid.to(torch.uint8).contiguous(), gt_ign.to(torch.uint8).contiguous()
    _lib.check(L.c3d_anchor_sample_finish(ptr(lab), ptr(max_ioa.contiguous()), ptr(idx), ptr(counts), ptr(best_idx.contiguous()),
                                          ptr(v8), ptr(i8), B, G, A, k, int(cap_pos), int(n_total), float(ignore_thresh),
                                          ptr(out), ptr(rng) if bump_rng else None, stream()))
    return out


def det_candidates(probs, boxes, prop_count, image_hw, score_thresh):
    """probs (B,P,K+1), boxes (B,P,K,4) fp32 -> cand_score (B,P*K) (-inf = filtered), cand_boxes (B,P*K,4) clipped,
    maxc (B,), total (B,) int32 (fast_rcnn.py:76-100 for the whole batch)."""
    L = _lib.lib()
    B, P, K1 = probs.shape
    K = K1 - 1
    dev = probs.device
    probs, boxes = probs.contiguous().float(), boxes.contiguous().float()
    cs = torch.empty((B, P * K), dtype=torch.float32, device=dev)
    cb = torch.empty((B, P * K, 4), dtype=torch.float32, device=dev)
    maxc = torch.empty((B,), dtype=torch.float32, device=dev)
    total = torch.empty((B,), dtype=torch.int32, device=dev)
    _lib.check(L.c3d_det_candidates(ptr(probs), ptr(boxes), ptr(prop_count.to(torch.int32).contiguous()),
                                    ptr(image_hw.contiguous().float()), B, P, K, float(score_thresh), ptr(cs), ptr(cb), ptr(maxc),
                                    ptr(total), stream()))
    return cs, cb, maxc, total


# ---- head losses (head_loss_ops.cu) -----------------------------------------------------------------------------------
def box_loss_fwd(pred, classes, valid, boxes, gt_boxes, K, weights):
    """pred (R, ld) fp32 rows [K+1 scores | 4K deltas | pad] -> acc (8,) fp32 [sum CE, sum L1(fg), #valid, #fg, #correct,
    #fg correct, #fg predicted background, 0] (fast_rcnn.py:145-194)."""
    L = _lib.lib()
    R, ld = pred.shape
    acc = torch.empty(8, dtype=torch.float32, device=pred.device)
    w = (f32 * 4)(*[float(v) for v in weights])
    _lib.check(L.c3d_box_loss_fwd(ptr(pred), ld, ptr(classes), ptr(valid), ptr(boxes), ptr(gt_boxes), R, int(K), w, ptr(acc), stream()))
    return acc


def box_loss_bwd(pred, classes, valid, boxes, gt_boxes, K, weights, acc, g2):
    L = _lib.lib()
    R, ld = pred.shape
    dpred = torch.empty_like(pred)
    w = (f32 * 4)(*[float(v) for v in weights])
    _lib.check(L.c3d_box_loss_bwd(ptr(pred), ld, ptr(classes), ptr(valid), ptr(boxes), ptr(gt_boxes), R, int(K), w, ptr(acc), ptr(g2),
                                  ptr(dpred), stream()))
    return dpred


def cube_gather(pred, classes, boxes, meta, priors, gt3, gtR, per_image, K, virtual_focal):
    """-> raw (n,13), aux (n,28): the inputs of c3d_cube_loss_fwd/bwd (roi_heads.py:372-461)."""
    L = _lib.lib()
    n, ld = pred.shape
    raw = torch.empty((n, 13), dtype=torch.float32, device=pred.device)
    aux = torch.empty((n, 28), dtype=torch.float32, device=pred.device)
    _lib.check(L.c3d_cube_gather(ptr(pred), ld, ptr(classes), ptr(boxes), ptr(meta), ptr(priors), ptr(gt3), ptr(gtR), n, int(per_image),
                                 int(K), float(virtual_focal), ptr(raw), ptr(aux), stream()))
    return raw, aux


def cube_reduce_fwd(rows, valid):
    L = _lib.lib()
    sums = torch.empty(12, dtype=torch.float32, device=rows.device)
    cnts = torch.empty(8, dtype=torch.float32, device=rows.device)
    _lib.check(L.c3d_cube_reduce_fwd(ptr(rows), ptr(valid), rows.shape[0], ptr(sums), ptr(cnts), stream()))
    return sums, cnts


def cube_reduce_bwd(rows, valid, cnts, g6):
    L = _lib.lib()
    n = rows.shape[0]
    d = torch.empty((n, 6), dtype=torch.float32, device=rows.device)
    _lib.check(L.c3d_cube_reduce_bwd(ptr(rows), ptr(valid), n, ptr(cnts), ptr(g6), ptr(d), stream()))
    return d


def cube_scatter(draw, classes, K, ld):
    L = _lib.lib()
    n = draw.shape[0]
    dpred = torch.empty((n, ld), dtype=torch.float32, device=draw.device)
    _lib.check(L.c3d_cube_scatter(ptr(draw), ptr(classes), n, int(K), int(ld), ptr(dpred), stream()))
    return dpred
