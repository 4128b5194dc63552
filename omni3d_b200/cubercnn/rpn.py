"""RPNWithIgnore on the accelerated path: batched, sync-free restatement of
cubercnn/modeling/proposal_generator/rpn.py:19-354 over detectron2's RPN / StandardRPNHead /
DefaultAnchorGenerator / find_top_rpn_proposals (SURVEY.md A.3).

All images of the batch are processed together (no per-image Python loop, no .item()/.tolist()):
  head      3x3 conv + ReLU and the two 1x1 predictors fused into one 16-channel fp32 conv (wgmma)
  labels    (B,G,A) IoU -> matcher [0.05] with low-quality matches, best-anchor override, ignore regions
  sampling  IoU-weighted sampling without replacement as batched Gumbel top-k on the device
  proposals decode, per-level top-k, clip, c3d_nms_batched (coordinate-trick offsets), top post_nms_topk
"""
import math

import torch
import torch.nn.functional as F
from torch import nn

from .. import kernels as Kx
from ..nnfunc import ConvBias
from .registry import PROPOSAL_GENERATOR_REGISTRY

SCALE_CLAMP = math.log(1000.0 / 16)


# ---- box utilities (fp32, any device) ------------------------------------------------------------
def box_area(b):
    return (b[..., 2] - b[..., 0]) * (b[..., 3] - b[..., 1])


def pairwise_inter(a, b):
    """a (B,G,4), b (B,P,4) or (P,4) -> (B,G,P) intersection areas."""
    if b.dim() == 2:
        b = b.unsqueeze(0)
    wh = torch.min(a[:, :, None, 2:], b[:, None, :, 2:]) - torch.max(a[:, :, None, :2], b[:, None, :, :2])
    wh = wh.clamp_(min=0)
    return wh[..., 0] * wh[..., 1]


def pairwise_iou(a, b):
    inter = pairwise_inter(a, b)
    bb = b.unsqueeze(0) if b.dim() == 2 else b
    union = box_area(a)[:, :, None] + box_area(bb)[:, None, :] - inter
    return torch.where(inter > 0, inter / union, torch.zeros((), dtype=inter.dtype, device=inter.device))


def pairwise_ioa(a, b):
    inter = pairwise_inter(a, b)
    bb = b.unsqueeze(0) if b.dim() == 2 else b
    return torch.where(inter > 0, inter / box_area(bb)[:, None, :], torch.zeros((), dtype=inter.dtype, device=inter.device))


def paired_iou(b1, b2):
    wh = (torch.min(b1[..., 2:], b2[..., 2:]) - torch.max(b1[..., :2], b2[..., :2])).clamp(min=0)
    inter = wh[..., 0] * wh[..., 1]
    return inter / (box_area(b1) + box_area(b2) - inter)


def get_deltas(src, tgt, weights):
    sw, sh = src[..., 2] - src[..., 0], src[..., 3] - src[..., 1]
    scx, scy = src[..., 0] + 0.5 * sw, src[..., 1] + 0.5 * sh
    tw, th = tgt[..., 2] - tgt[..., 0], tgt[..., 3] - tgt[..., 1]
    tcx, tcy = tgt[..., 0] + 0.5 * tw, tgt[..., 1] + 0.5 * th
    wx, wy, ww, wh = weights
    return torch.stack((wx * (tcx - scx) / sw, wy * (tcy - scy) / sh, ww * torch.log(tw / sw), wh * torch.log(th / sh)), -1)


def apply_deltas(deltas, boxes, weights):
    """deltas (...,4k), boxes (...,4) -> (...,4k)."""
    deltas = deltas.float()
    w, h = boxes[..., 2] - boxes[..., 0], boxes[..., 3] - boxes[..., 1]
    cx, cy = boxes[..., 0] + 0.5 * w, boxes[..., 1] + 0.5 * h
    wx, wy, ww, wh = weights
    dx, dy = deltas[..., 0::4] / wx, deltas[..., 1::4] / wy
    dw = torch.clamp(deltas[..., 2::4] / ww, max=SCALE_CLAMP)
    dh = torch.clamp(deltas[..., 3::4] / wh, max=SCALE_CLAMP)
    pcx, pcy = dx * w[..., None] + cx[..., None], dy * h[..., None] + cy[..., None]
    pw, ph = torch.exp(dw) * w[..., None], torch.exp(dh) * h[..., None]
    out = torch.stack((pcx - 0.5 * pw, pcy - 0.5 * ph, pcx + 0.5 * pw, pcy + 0.5 * ph), dim=-1)
    return out.reshape(deltas.shape)


def gumbel_topk_sample(weights, k, generator=None):
    """Weighted sampling WITHOUT replacement of up to k items per row (Efraimidis-Spirakis / Gumbel top-k):
    equivalent in distribution to torch.multinomial(weights, n, replacement=False) used at rpn.py:317-324, but
    batched and sync-free.  weights (B,N) >= 0 (0 = not a candidate) -> idx (B,k), valid (B,k) bool."""
    u = torch.rand(weights.shape, device=weights.device, generator=generator).clamp_(min=1e-20)
    keys = torch.log(weights.clamp(min=0)) - torch.log(-torch.log(u))
    keys = torch.where(weights > 0, keys, torch.full_like(keys, -float("inf")))
    k = min(k, weights.shape[1])
    val, idx = keys.topk(k, dim=1)
    return idx, torch.isfinite(val)


class AnchorGenerator:
    """DefaultAnchorGenerator: sizes one per level, ratios (0.5,1,2); anchor index (y*W + x)*A + a."""

    def __init__(self, sizes, ratios, strides, offset=0.0):
        n = len(strides)
        sizes = list(sizes) * n if len(sizes) == 1 else list(sizes)
        ratios = list(ratios) * n if len(ratios) == 1 else list(ratios)
        self.strides, self.offset = strides, offset
        self.cell = []
        for s_l, r_l in zip(sizes, ratios):
            a = []
            for size in s_l:
                area = size ** 2.0
                for r in r_l:
                    w = math.sqrt(area / r)
                    h = r * w
                    a.append([-w / 2.0, -h / 2.0, w / 2.0, h / 2.0])
            self.cell.append(torch.tensor(a))
        self.num_anchors = len(self.cell[0])
        self._cache = {}

    def __call__(self, shapes, device):
        key = (tuple(shapes), str(device))
        if key not in self._cache:
            out = []
            for (gh, gw), stride, base in zip(shapes, self.strides, self.cell):
                sx = torch.arange(self.offset * stride, gw * stride, step=stride, dtype=torch.float32, device=device)
                sy = torch.arange(self.offset * stride, gh * stride, step=stride, dtype=torch.float32, device=device)
                yy, xx = torch.meshgrid(sy, sx, indexing="ij")
                sh = torch.stack((xx.reshape(-1), yy.reshape(-1), xx.reshape(-1), yy.reshape(-1)), dim=1)
                out.append((sh.view(-1, 1, 4) + base.to(device).view(1, -1, 4)).reshape(-1, 4))
            self._cache[key] = out
        return self._cache[key]


class StandardRPNHead(nn.Module):
    def __init__(self, in_channels, num_anchors):
        super().__init__()
        self.conv = nn.Conv2d(in_channels, in_channels, 3, padding=1)
        self.objectness_logits = nn.Conv2d(in_channels, num_anchors, 1)
        self.anchor_deltas = nn.Conv2d(in_channels, num_anchors * 4, 1)
        for l in (self.conv, self.objectness_logits, self.anchor_deltas):
            nn.init.normal_(l.weight, std=0.01)
            nn.init.constant_(l.bias, 0)
        self.A = num_anchors

    def forward(self, feats):
        A = self.A
        pad = 16 - 5 * A
        w = torch.cat([self.objectness_logits.weight, self.anchor_deltas.weight,
                       self.conv.weight.new_zeros((pad,) + tuple(self.anchor_deltas.weight.shape[1:]))], 0)
        b = torch.cat([self.objectness_logits.bias, self.anchor_deltas.bias, self.conv.bias.new_zeros(pad)], 0)
        logits, deltas = [], []
        for x in feats:
            t = ConvBias.apply(x, self.conv.weight, self.conv.bias, None, 1, 1, True, False)
            o = ConvBias.apply(t, w, b, None, 1, 0, False, True)            # (N,H,W,16) fp32
            N = o.shape[0]
            logits.append(o[..., :A].reshape(N, -1))
            deltas.append(o[..., A:5 * A].reshape(N, -1, 4))
        return logits, deltas


@PROPOSAL_GENERATOR_REGISTRY.register()
class RPNWithIgnore(nn.Module):
    def __init__(self, cfg, in_channels, strides):
        super().__init__()
        R = cfg.MODEL.RPN
        if R.OBJECTNESS_UNCERTAINTY.lower() != "iouness":
            raise NotImplementedError("accelerated path covers OBJECTNESS_UNCERTAINTY 'IoUness' (Base.yaml:56)")
        if R.HEAD_NAME != "StandardRPNHead" or list(R.IOU_LABELS) != [0, -1, 1]:
            raise NotImplementedError("RPN head / IOU_LABELS variant not on the accelerated path")
        self.in_features = list(R.IN_FEATURES)
        self.strides = [strides[f] for f in self.in_features]
        self.anchor_generator = AnchorGenerator(cfg.MODEL.ANCHOR_GENERATOR.SIZES, cfg.MODEL.ANCHOR_GENERATOR.ASPECT_RATIOS,
                                                self.strides, cfg.MODEL.ANCHOR_GENERATOR.OFFSET)
        self.rpn_head = StandardRPNHead(in_channels, self.anchor_generator.num_anchors)
        self.iou_thresholds = list(R.IOU_THRESHOLDS)
        if self.iou_thresholds[0] != self.iou_thresholds[-1]:
            # a real ignore band [lo, hi) (detectron2 default [0.3, 0.7]) would need label -1 between the thresholds;
            # the accelerated matcher implements the reference's single-threshold form (Base.yaml:57: [0.05, 0.05])
            raise NotImplementedError("RPN.IOU_THRESHOLDS with lo != hi (ignore band) is not on the accelerated path")
        self.batch_size_per_image = R.BATCH_SIZE_PER_IMAGE
        self.positive_fraction = R.POSITIVE_FRACTION
        self.pre_nms_topk = {True: R.PRE_NMS_TOPK_TRAIN, False: R.PRE_NMS_TOPK_TEST}
        self.post_nms_topk = {True: R.POST_NMS_TOPK_TRAIN, False: R.POST_NMS_TOPK_TEST}
        self.nms_thresh = R.NMS_THRESH
        self.min_box_size = float(cfg.MODEL.PROPOSAL_GENERATOR.MIN_SIZE)
        self.weights = tuple(R.BBOX_REG_WEIGHTS)
        self.ignore_thresh = R.IGNORE_THRESHOLD
        self.generator = None          # optional torch.Generator for the sampling noise
        # torchvision.ops.batched_nms switches from the coordinate trick to per-category NMS above this many
        # box coordinates (20000 on CUDA, 4000 on CPU); the reference runs on CUDA.
        self.nms_trick_max_numel = 20000
        self.fused_loss = True                 # c3d_rpn_loss_fwd/bwd instead of the (B,A)-shaped torch formulation
        self.fused_decode = True               # c3d_rpn_decode_level instead of ~35 torch ops per level
        self.fused_topk = True                 # c3d_topk_segments instead of ATen topk per level + radix sort
        self.fused_sampling = True             # c3d_anchor_sample_* instead of the torch Gumbel top-k formulation
        self.stats = {}

    # -- labels -----------------------------------------------------------------------------------
    @torch.no_grad()
    def match_anchors(self, anchors, gt_boxes, gt_valid, gt_ign=None):
        """anchors (A,4); gt_boxes (B,G,4) padded; gt_valid (B,G) bool (valid & not ignore); gt_ign (B,G) ignore regions.
        -> matched_idx (B,A), matched_iou (B,A), labels (B,A) int8 in {0,1}, best (B,A) bool, max IoA with ignore
        regions (B,A).  CUDA: two c3d_anchor_match passes; CPU (host-logic tests): the same formulas in torch."""
        if gt_ign is None:
            gt_ign = torch.zeros_like(gt_valid)
        lo = self.iou_thresholds[-1]
        if anchors.is_cuda:
            from .. import kernels as Kx
            idx, vals, labels, ioa, best_idx = Kx.anchor_match(anchors, gt_boxes, gt_valid, gt_ign, lo)
            A = anchors.shape[0]
            best = torch.zeros(labels.shape, dtype=torch.int32, device=labels.device)
            best.scatter_add_(1, best_idx.clamp(max=A - 1).long(), gt_valid.to(torch.int32))
            return idx, vals, labels, (best > 0) & (labels == 1), ioa
        iou = pairwise_iou(gt_boxes, anchors)                                   # (B,G,A)
        iou = torch.where(gt_valid[:, :, None], iou, torch.full_like(iou, -1.0))
        vals, idx = iou.max(dim=1)
        labels = (vals >= lo).to(torch.int8)
        rowmax = iou.max(dim=2, keepdim=True).values                            # best IoU of every GT
        lowq = ((iou == rowmax) & gt_valid[:, :, None]).any(dim=1)              # allow_low_quality_matches
        labels = torch.where(lowq, torch.ones_like(labels), labels)
        # the arg-max anchor of every valid GT, kept positive after sampling if the matcher said positive
        best_idx = iou.argmax(dim=2)                                            # (B,G)
        best = torch.zeros(labels.shape, dtype=torch.int32, device=labels.device)
        best.scatter_add_(1, best_idx, gt_valid.to(torch.int32))
        best = (best > 0) & (labels == 1)
        ioa = pairwise_ioa(gt_boxes, anchors)                                    # (B,G,A)
        ioa = torch.where(gt_ign[:, :, None], ioa, torch.zeros_like(ioa)).max(dim=1).values
        return idx, vals.clamp(min=0), labels, best, ioa

    @torch.no_grad()
    def label_and_sample_anchors(self, anchors, gt_boxes, gt_classes, gt_present):
        """gt_classes (B,G) (-1 = ignore region), gt_present (B,G) bool (non-padding)."""
        valid = gt_present & (gt_classes >= 0)
        ign = gt_present & (gt_classes < 0)
        if anchors.is_cuda and self.fused_sampling and self.generator is None:
            idx, miou, lab, ioa, best_idx = Kx.anchor_match(anchors, gt_boxes, valid, ign, self.iou_thresholds[-1])
            out = Kx.anchor_sample(lab, miou, ioa, best_idx, valid, ign, self.batch_size_per_image,
                                   int(self.batch_size_per_image * self.positive_fraction), self.ignore_thresh)
            return out, idx
        idx, miou, lab, best, ioa = self.match_anchors(anchors, gt_boxes, valid, ign)
        B, A = lab.shape
        n_total = self.batch_size_per_image
        cap_pos = int(n_total * self.positive_fraction)
        pos_c, neg_c = lab == 1, lab == 0
        num_pos = pos_c.sum(1).clamp(max=cap_pos)
        num_neg = torch.minimum(neg_c.sum(1), n_total - num_pos)
        w = miou + 1e-4
        p_idx, p_ok = gumbel_topk_sample(torch.where(pos_c, w, torch.zeros_like(w)), cap_pos, self.generator)
        n_idx, n_ok = gumbel_topk_sample(torch.where(neg_c, w, torch.zeros_like(w)), n_total, self.generator)
        ar_p = torch.arange(p_idx.shape[1], device=lab.device)[None]
        ar_n = torch.arange(n_idx.shape[1], device=lab.device)[None]
        out = torch.full_like(lab, -1)
        # scatter with masks (invalid picks are routed to a dummy column)
        dummy = torch.full((B, 1), -1, dtype=out.dtype, device=out.device)
        ext = torch.cat([out, dummy], 1)
        n_sel = n_ok & (ar_n < num_neg[:, None])
        p_sel = p_ok & (ar_p < num_pos[:, None])
        ext.scatter_(1, torch.where(n_sel, n_idx, torch.full_like(n_idx, A)), torch.zeros_like(n_idx, dtype=out.dtype))
        ext.scatter_(1, torch.where(p_sel, p_idx, torch.full_like(p_idx, A)), torch.ones_like(p_idx, dtype=out.dtype))
        out = ext[:, :A].contiguous()
        out[best] = 1
        return self.finish_labels(out, anchors, gt_boxes, ign, ioa), idx

    @torch.no_grad()
    def finish_labels(self, labels, anchors, gt_boxes, ign, ioa=None):
        """background anchors lying >= IGNORE_THRESHOLD inside an ignore box become -1 (rpn.py:93-105;
        only when the image has more than one background anchor, as there)."""
        if ioa is None:
            ioa = pairwise_ioa(gt_boxes, anchors)                                # (B,G,A)
            ioa = torch.where(ign[:, :, None], ioa, torch.zeros_like(ioa)).max(dim=1).values
        bg = labels == 0
        hit = bg & (ioa >= self.ignore_thresh) & (bg.sum(1, keepdim=True) > 1) & ign.any(1, keepdim=True)
        return torch.where(hit, torch.full_like(labels, -1), labels)

    # -- losses -----------------------------------------------------------------------------------
    def losses(self, anchors, logits, deltas, labels, matched_idx, gt_boxes):
        B = labels.shape[0]
        norm = self.batch_size_per_image * B
        if logits.is_cuda and self.fused_loss:
            from ..nnfunc import RPNLossSums
            acc = RPNLossSums.apply(logits, deltas, labels, matched_idx, gt_boxes, anchors, self.weights)
            with torch.no_grad():
                a = acc.detach()
                npos, rest = a[2], labels.numel() - a[2]
                self.stats = {"rpn/num_pos_anchors": npos / B, "rpn/num_neg_anchors": a[3] / B,
                              "rpn/conf_pos_anchors": a[4] / npos.clamp(min=1), "rpn/conf_neg_anchors": a[5] / rest.clamp(min=1)}
            return {"rpn/cls": acc[0] / norm, "rpn/loc": acc[1] / norm}
        pos = labels == 1
        matched = torch.gather(gt_boxes, 1, matched_idx[:, :, None].expand(-1, -1, 4))       # (B,A,4)
        a = anchors.unsqueeze(0).expand(B, -1, -1)
        target = paired_iou(a, matched).detach()
        posf = pos.float()
        tgt = torch.where(pos, target, torch.zeros_like(target))
        bce = F.binary_cross_entropy_with_logits(logits, tgt, reduction="none")
        loss_cls = (bce * tgt * posf).sum()
        gt_d = get_deltas(a, matched, self.weights)
        l1 = (deltas - gt_d).abs().sum(-1)
        loss_loc = (torch.where(pos, l1 * target, torch.zeros_like(l1))).sum()
        norm = self.batch_size_per_image * B
        with torch.no_grad():
            sig = torch.sigmoid(logits)
            npos = posf.sum()
            self.stats = {"rpn/num_pos_anchors": npos / B, "rpn/num_neg_anchors": (labels == 0).float().sum() / B,
                          "rpn/conf_pos_anchors": (sig * posf).sum() / npos.clamp(min=1),
                          "rpn/conf_neg_anchors": (sig * (1 - posf)).sum() / (posf.numel() - npos).clamp(min=1)}
        return {"rpn/cls": loss_cls / norm, "rpn/loc": loss_loc / norm}

    # -- proposals --------------------------------------------------------------------------------
    @torch.no_grad()
    def predict_proposals(self, anchors_per_level, logits_per_level, deltas_per_level, image_sizes, sizes_dev=None):
        """-> boxes (B,post,4), logits (B,post), count (B,) int32; slots >= count are padding (score -inf)."""
        training = self.training
        B = logits_per_level[0].shape[0]
        dev = logits_per_level[0].device
        hw = sizes_dev if sizes_dev is not None else torch.as_tensor(image_sizes, dtype=torch.float32, device=dev)  # (B,2) = (h,w)
        ks = [min(lg.shape[1], self.pre_nms_topk[training]) for lg in logits_per_level]
        if dev.type == "cuda" and self.fused_decode:
            # one c3d_rpn_decode_level launch per level: apply_deltas + clip + finite/min-size filter, straight into the
            # concatenated candidate arrays (plus per-image valid count and max kept coordinate)
            Ktot = sum(ks)
            boxes = torch.empty((B, Ktot, 4), device=dev)
            key = torch.empty((B, Ktot), device=dev)
            lvl = torch.empty((B, Ktot), device=dev)
            nvalid = torch.zeros((B,), dtype=torch.int32, device=dev)
            maxc = torch.zeros((B,), device=dev)
            hw = hw.contiguous().float()
            col = 0
            if self.fused_topk:       # all levels' pre-NMS top-k in ONE launch (c3d_topk_segments), then the score sort
                tv, ti = Kx.topk_segments([(lg if lg.stride(1) == 1 else lg.contiguous(), k)
                                           for lg, k in zip(logits_per_level, ks)], want_idx64=True)
            for li, (anc, lg, dl, k) in enumerate(zip(anchors_per_level, logits_per_level, deltas_per_level, ks)):
                if self.fused_topk:
                    s, i = tv[:, col:col + k], ti[:, col:col + k]
                else:
                    s, i = lg.topk(k, dim=1)
                Kx.rpn_decode_level(i, s, dl.contiguous(), anc, hw, self.weights, SCALE_CLAMP, self.min_box_size, li, col,
                                    boxes, key, lvl, nvalid, maxc)
                col += k
            if self.fused_topk and Ktot <= 8192:
                key, order = Kx.topk_segments([(key, Ktot)], want_idx64=True)
            else:
                key, order = key.sort(dim=1, descending=True)
            boxes = torch.gather(boxes, 1, order[:, :, None].expand(-1, -1, 4))
            lvl = torch.gather(lvl, 1, order)
        else:
            cand_b, cand_s, cand_l = [], [], []
            for li, (anc, lg, dl, k) in enumerate(zip(anchors_per_level, logits_per_level, deltas_per_level, ks)):
                s, i = lg.topk(k, dim=1)
                d = torch.gather(dl, 1, i[:, :, None].expand(-1, -1, 4))
                cand_b.append(apply_deltas(d, anc[i], self.weights))
                cand_s.append(s)
                cand_l.append(torch.full((k,), li, dtype=torch.float32, device=dev))
            boxes, scores = torch.cat(cand_b, 1), torch.cat(cand_s, 1)
            lvl = torch.cat(cand_l)[None].expand(B, -1)
            lim = torch.stack((hw[:, 1], hw[:, 0], hw[:, 1], hw[:, 0]), 1)[:, None, :]
            finite = torch.isfinite(boxes).all(-1) & torch.isfinite(scores)
            boxes = torch.minimum(boxes.clamp(min=0), lim)
            keep = finite & ((boxes[..., 2] - boxes[..., 0]) > self.min_box_size) & \
                ((boxes[..., 3] - boxes[..., 1]) > self.min_box_size)
            key = torch.where(keep, scores, torch.full_like(scores, -float("inf")))
            key, order = key.sort(dim=1, descending=True)
            boxes = torch.gather(boxes, 1, order[:, :, None].expand(-1, -1, 4))
            lvl = torch.gather(lvl, 1, order)
            nvalid = keep.sum(1).to(torch.int32)
            keep_sorted = torch.gather(keep, 1, order)
            maxc = torch.where(keep_sorted[:, :, None], boxes, torch.full_like(boxes, -float("inf"))).amax(dim=(1, 2))
        # torchvision batched_nms: per-level NMS; for small inputs it uses the "coordinate trick" (shift every
        # level by level * (max coordinate + 1)) — the kernel reproduces either form per image.
        post = self.post_nms_topk[training]
        kidx, kcnt = Kx.nms_batched(boxes, nvalid, self.nms_thresh, post, cats=lvl.contiguous(), maxc=maxc,
                                    trick_max_numel=self.nms_trick_max_numel, ncat=len(anchors_per_level),
                                    max_per_cat=self.pre_nms_topk[training])
        safe = kidx.clamp(min=0).long()
        out_b = torch.gather(boxes, 1, safe[:, :, None].expand(-1, -1, 4))
        out_s = torch.gather(key, 1, safe)
        pad = kidx < 0
        out_b = torch.where(pad[:, :, None], torch.zeros_like(out_b), out_b)
        out_s = torch.where(pad, torch.full_like(out_s, -float("inf")), out_s)
        return out_b, out_s, kcnt

    def forward(self, features, image_sizes, gt=None, sizes_dev=None):
        feats = [features[f] for f in self.in_features]
        shapes = [tuple(f.shape[1:3]) for f in feats]
        anchors_l = self.anchor_generator(shapes, feats[0].device)
        logits_l, deltas_l = self.rpn_head(feats)
        losses = {}
        if self.training:
            anchors = torch.cat(anchors_l, 0)
            logits, deltas = torch.cat(logits_l, 1), torch.cat(deltas_l, 1)
            if gt.get("anchor_labels") is not None:           # parity tests inject the oracle's sampled labels
                labels = gt["anchor_labels"]
                valid = gt["present"] & (gt["classes"] >= 0)
                idx = self.match_anchors(anchors, gt["boxes"], valid)[0]
            else:
                labels, idx = self.label_and_sample_anchors(anchors, gt["boxes"], gt["classes"], gt["present"])
            losses = self.losses(anchors, logits, deltas, labels, idx, gt["boxes"])
        if gt is not None and gt.get("proposals") is not None:   # parity tests inject the oracle's proposals
            props = gt["proposals"]
        else:
            props = self.predict_proposals(anchors_l, [l.detach() for l in logits_l], [d.detach() for d in deltas_l],
                                           image_sizes, sizes_dev)
        return props, losses
