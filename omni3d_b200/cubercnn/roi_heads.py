"""ROIHeads3D + FastRCNNOutputs + CubeHead on the accelerated path — batched, sync-free restatement of
cubercnn/modeling/roi_heads/{roi_heads.py:39-941, fast_rcnn.py:16-260, cube_head.py:19-202} over
detectron2's StandardROIHeads / ROIPooler / FastRCNNConvFCHead / FastRCNNOutputLayers (SURVEY.md A.4).

Fixed-shape tensors replace per-image Instances lists: every image contributes exactly
BATCH_SIZE_PER_IMAGE sampled-proposal slots and POSITIVE_FRACTION*BATCH_SIZE foreground slots (masked
when fewer exist), so the whole head runs without host synchronisation.  ROIAlign runs on libc3d.so, the
FC stacks are plain bf16 library GEMMs (cuBLAS through torch, as the task allows for plain GEMMs).
"""
import math

import torch
import torch.nn.functional as F
from torch import nn

from ..nnfunc import BoxLoss, CubeHeadLoss, LinearAct, ROIAlign, TwoHeadFC1
from . import geometry as G
from .registry import ROI_CUBE_HEAD_REGISTRY, ROI_HEADS_REGISTRY
from .rpn import apply_deltas, get_deltas, gumbel_topk_sample, pairwise_ioa, pairwise_iou

SQRT2 = 1.41421356


def assign_levels(boxes, min_level=2, max_level=6):
    size = torch.sqrt(((boxes[..., 2] - boxes[..., 0]) * (boxes[..., 3] - boxes[..., 1])).clamp(min=0))
    lvl = torch.floor(4 + torch.log2(size / 224 + 1e-8))
    return lvl.clamp(min=min_level, max=max_level) - min_level


def fc(x, lin, relu=False, chw=None, out_fp32=False):
    """[relu](x W^T + b) on the wgmma GEMM (c3d_linear_*).  chw = (C, P*P): W is the reference's weight over a
    (C,P,P)-flattened RoI while x is the (P,P,C)-flattened NHWC RoI the ROIAlign kernel emits (features re-ordered
    when the weight is packed to bf16; the weight gradient is written back in the master's order)."""
    return LinearAct.apply(x, lin.weight, lin.bias, relu, out_fp32, chw)


_zero_pad = {}


def fused_predictors(h, lins, n_pad, split=True):
    """several small nn.Linear predictors over the same features as ONE zero-padded GEMM -> list of fp32 outputs
    (split=False: the padded (rows, n_pad) fp32 output itself, columns in the order of `lins`)."""
    widths = [l.weight.shape[0] for l in lins]
    pad = n_pad - sum(widths)
    key = (pad, h.shape[1], h.device)
    z = _zero_pad.get(key)
    if z is None:
        z = _zero_pad[key] = (torch.zeros((pad, h.shape[1]), device=h.device), torch.zeros(pad, device=h.device))
    w = torch.cat([l.weight for l in lins] + [z[0]], 0)
    b = torch.cat([l.bias for l in lins] + [z[1]], 0)
    y = LinearAct.apply(h, w, b, False, True, None)
    if not split:
        return y
    out, o = [], 0
    for n in widths:
        out.append(y[:, o:o + n])
        o += n
    return out


class FastRCNNConvFCHead(nn.Sequential):
    def __init__(self, in_dim, fc_dims):
        super().__init__()
        self.add_module("flatten", nn.Flatten())
        d = in_dim
        for k, fc_dim in enumerate(fc_dims):
            fc = nn.Linear(d, fc_dim)
            self.add_module("fc%d" % (k + 1), fc)
            self.add_module("fc_relu%d" % (k + 1), nn.ReLU())
            d = fc_dim
        for k in range(len(fc_dims)):
            fc = getattr(self, "fc%d" % (k + 1))
            nn.init.kaiming_uniform_(fc.weight, a=1)
            nn.init.constant_(fc.bias, 0)
        self.out_dim = d


class FastRCNNOutputs(nn.Module):
    def __init__(self, in_dim, num_classes):
        super().__init__()
        self.cls_score = nn.Linear(in_dim, num_classes + 1)
        self.bbox_pred = nn.Linear(in_dim, num_classes * 4)
        nn.init.normal_(self.cls_score.weight, std=0.01)
        nn.init.normal_(self.bbox_pred.weight, std=0.001)
        for l in (self.cls_score, self.bbox_pred):
            nn.init.constant_(l.bias, 0)


@ROI_CUBE_HEAD_REGISTRY.register()
class CubeHead(nn.Module):
    def __init__(self, cfg, in_dim):
        super().__init__()
        H = cfg.MODEL.ROI_CUBE_HEAD
        if not (H.SHARED_FC and H.POSE_TYPE == "6d" and H.CLUSTER_BINS == 1 and H.NUM_CONV == 0 and H.USE_CONFIDENCE > 0):
            raise NotImplementedError("accelerated CubeHead covers SHARED_FC / 6d pose / no clusters / confidence on")
        K = self.num_classes = cfg.MODEL.ROI_HEADS.NUM_CLASSES
        self.feature_generator = nn.Sequential()
        d = in_dim
        for k in range(H.NUM_FC):
            fc = nn.Linear(d, H.FC_DIM)
            nn.init.kaiming_uniform_(fc.weight, a=1)
            nn.init.constant_(fc.bias, 0)
            self.feature_generator.add_module("fc%d" % (k + 1), fc)
            self.feature_generator.add_module("fc_relu%d" % (k + 1), nn.ReLU())
            d = H.FC_DIM
        for name, mult, bias in (("bbox_3D_dims", 3, 0), ("bbox_3D_center_deltas", 2, 0), ("bbox_3D_pose", 6, 0),
                                 ("bbox_3D_center_depth", 1, 0), ("bbox_3D_uncertainty", 1, 5)):
            lin = nn.Linear(d, K * mult)
            nn.init.normal_(lin.weight, std=0.001)
            nn.init.constant_(lin.bias, bias)
            setattr(self, name, lin)


@ROI_HEADS_REGISTRY.register()
class ROIHeads3D(nn.Module):
    def __init__(self, cfg, in_channels, strides, priors=None):
        super().__init__()
        RH, BH, H = cfg.MODEL.ROI_HEADS, cfg.MODEL.ROI_BOX_HEAD, cfg.MODEL.ROI_CUBE_HEAD
        ok = (H.DISENTANGLED_LOSS and H.CHAMFER_POSE and H.ALLOCENTRIC_POSE and H.VIRTUAL_DEPTH and H.Z_TYPE == "direct"
              and H.DIMS_PRIORS_ENABLED and H.DIMS_PRIORS_FUNC == "exp" and not H.INVERSE_Z_WEIGHT
              and H.SCALE_ROI_BOXES == 0.0 and H.LOSS_W_3D > 0 and H.LOSS_W_JOINT > 0 and BH.NUM_CONV == 0
              and BH.NAME == "FastRCNNConvFCHead" and BH.POOLER_TYPE == "ROIAlignV2" and not BH.CLS_AGNOSTIC_BBOX_REG
              and list(RH.IOU_LABELS) == [0, 1])
        if not ok:
            raise NotImplementedError("accelerated ROIHeads3D covers the BASELINE configuration (Base.yaml:61-86)")
        self.in_features = list(RH.IN_FEATURES)
        self.strides = [strides[f] for f in self.in_features]
        self.num_classes = K = RH.NUM_CLASSES
        self.batch_size_per_image = RH.BATCH_SIZE_PER_IMAGE
        self.positive_fraction = RH.POSITIVE_FRACTION
        self.iou_thresh = RH.IOU_THRESHOLDS[0]
        self.append_gt = RH.PROPOSAL_APPEND_GT
        self.pooled = BH.POOLER_RESOLUTION
        self.box_weights = tuple(BH.BBOX_REG_WEIGHTS)
        self.test_score_thresh, self.test_nms_thresh = RH.SCORE_THRESH_TEST, RH.NMS_THRESH_TEST
        self.test_topk = cfg.TEST.DETECTIONS_PER_IMAGE
        self.ignore_thresh = cfg.MODEL.RPN.IGNORE_THRESHOLD
        self.virtual_focal = H.VIRTUAL_FOCAL
        self.w = dict(w3d=H.LOSS_W_3D, xy=H.LOSS_W_XY, z=H.LOSS_W_Z, dims=H.LOSS_W_DIMS, pose=H.LOSS_W_POSE,
                      joint=H.LOSS_W_JOINT, conf=H.USE_CONFIDENCE)
        in_dim = in_channels * self.pooled * self.pooled
        self.in_channels = in_channels
        # construction order mirrors the reference (same-seed init): box head, predictor, 2nd predictor, cube head
        self.box_head = FastRCNNConvFCHead(in_dim, [BH.FC_DIM] * BH.NUM_FC)
        FastRCNNOutputs(self.box_head.out_dim, K)                 # RNG parity with roi_heads.py:151
        self.box_predictor = FastRCNNOutputs(self.box_head.out_dim, K)
        assert H.POOLER_RESOLUTION == self.pooled
        # same ROIAlign for both heads (Base.yaml:66-68,78-80): the cube head's RoIs are a prefix of the box head's sampled
        # RoIs, so its pooled features are a slice of the box head's instead of a second ROIAlign forward + backward
        self.share_pool = (H.POOLER_SAMPLING_RATIO == BH.POOLER_SAMPLING_RATIO and H.POOLER_TYPE == BH.POOLER_TYPE)
        self.cube_head = CubeHead(cfg, in_dim)
        if priors is not None:
            self.priors_dims_per_cat = nn.Parameter(torch.FloatTensor(priors["priors_dims_per_cat"]).unsqueeze(0))
        else:
            self.priors_dims_per_cat = nn.Parameter(torch.ones(1, K, 2, 3))
        self.priors_z_scales = nn.Parameter(torch.ones(K, H.CLUSTER_BINS))
        self.generator = None
        self.stats = {}
        self.fused_cube = True        # c3d_cube_loss_fwd/bwd; False = the batched torch fp32 formulation below
        self.fused_sampling = True    # c3d_label_sample_proposals; False = the batched torch formulation below
        self.fused_head_losses = True  # c3d_box_loss_* / c3d_cube_gather|reduce|scatter; False = the torch loss assembly
        # torchvision.ops.batched_nms: coordinate trick up to this many box coordinates, per-class NMS above (CUDA value)
        self.nms_trick_max_numel = 20000

    # -- proposal labelling / sampling (roi_heads.py:826-929) -----------------------------------------
    @torch.no_grad()
    def match_proposals(self, boxes, pvalid, gt):
        """boxes (B,P,4), pvalid (B,P) -> matched gt idx (B,P), iou (B,P), class label (B,P) with K = background,
        -1 = ignore/invalid."""
        K = self.num_classes
        valid = gt["present"] & (gt["classes"] >= 0)
        ign = gt["present"] & (gt["classes"] < 0)
        iou = pairwise_iou(gt["boxes"], boxes)
        iou = torch.where(valid[:, :, None], iou, torch.full_like(iou, -1.0))
        vals, idx = iou.max(dim=1)
        fg = vals >= self.iou_thresh
        ioa = pairwise_ioa(gt["boxes"], boxes)
        ioa = torch.where(ign[:, :, None], ioa, torch.zeros_like(ioa)).max(dim=1).values
        bg = ~fg & pvalid                     # roi_heads.py:892-897: the rule needs > 1 REAL background proposals ...
        ign_hit = (bg & (ioa >= self.ignore_thresh) & (bg.sum(1, keepdim=True) > 1) & ign.any(1, keepdim=True)
                   & valid.any(1, keepdim=True))       # ... and is dropped when the image has no valid GT (:846-855)
        cls = torch.gather(gt["classes"], 1, idx)
        cls = torch.where(fg, cls, torch.full_like(cls, K))
        cls = torch.where(ign_hit | ~pvalid, torch.full_like(cls, -1), cls)
        return idx, vals.clamp(min=0), cls

    @torch.no_grad()
    def label_and_sample_proposals(self, prop_boxes, prop_count, gt):
        """-> dict of fixed-shape (B,S,...) sampled tensors; fg samples occupy the first F slots."""
        if gt.get("sampled") is not None:                     # parity tests inject the oracle's sampled set
            return gt["sampled"]
        B, P, _ = prop_boxes.shape
        dev = prop_boxes.device
        S, K = self.batch_size_per_image, self.num_classes
        G = gt["boxes"].shape[1]
        if (dev.type == "cuda" and self.fused_sampling and self.generator is None and G <= 256
                and P + (G if self.append_gt else 0) <= 2048):
            # one launch: matcher + ignore rule + IoU-weighted sampling + fg-first compaction + GT gather
            from .. import kernels as Kx
            out = Kx.label_sample_proposals(prop_boxes, prop_count, gt, K, S, int(S * self.positive_fraction), self.iou_thresh,
                                            self.ignore_thresh, append_gt=self.append_gt)
            st = out.pop("stats")
            self.stats["roi_head/num_fg_samples"] = st[0] / B
            self.stats["roi_head/num_bg_samples"] = st[1] / B
            out["fcap"] = int(S * self.positive_fraction)
            return out
        pvalid = torch.arange(P, device=dev)[None] < prop_count[:, None]
        boxes = prop_boxes
        if self.append_gt:
            gvalid = gt["present"] & (gt["classes"] >= 0)
            boxes = torch.cat([prop_boxes, gt["boxes"]], 1)
            pvalid = torch.cat([pvalid, gvalid], 1)
        S, K = self.batch_size_per_image, self.num_classes
        Fcap = int(S * self.positive_fraction)
        if True:
            midx, miou, cls = self.match_proposals(boxes, pvalid, gt)
            fg_c, bg_c = (cls >= 0) & (cls < K), cls == K
            w = miou + 1e-4
            num_fg = fg_c.sum(1).clamp(max=Fcap)
            num_bg = torch.minimum(bg_c.sum(1), S - num_fg)
            f_idx, f_ok = gumbel_topk_sample(torch.where(fg_c, w, torch.zeros_like(w)), Fcap, self.generator)
            b_idx, b_ok = gumbel_topk_sample(torch.where(bg_c, w, torch.zeros_like(w)), S, self.generator)
            f_ok &= torch.arange(f_idx.shape[1], device=dev)[None] < num_fg[:, None]
            # background picks fill slots Fcap.. (S - Fcap of them, plus unused fg capacity at the tail)
            b_take = torch.arange(b_idx.shape[1], device=dev)[None] < num_bg[:, None]
            b_ok &= b_take
            # [fg picks | bg picks] compacted (stable) to exactly S slots: valid fg first, then valid bg
            sel = torch.cat([f_idx, b_idx], 1)
            sel_ok = torch.cat([f_ok, b_ok], 1)
            pos = torch.arange(sel.shape[1], device=dev)[None] + (~sel_ok).long() * (10 * sel.shape[1])
            order = pos.argsort(dim=1)[:, :S]
            sel, sel_ok = torch.gather(sel, 1, order), torch.gather(sel_ok, 1, order)
            bsel = torch.gather(boxes, 1, sel[:, :, None].expand(-1, -1, 4))
            cls_sel = torch.where(sel_ok, torch.gather(cls, 1, sel), torch.full_like(sel, -1))
            midx_sel = torch.gather(midx, 1, sel)
        g = lambda t: torch.gather(t, 1, midx_sel.reshape(B, -1, *([1] * (t.dim() - 2))).expand(-1, -1, *t.shape[2:]))
        out = dict(boxes=bsel, valid=sel_ok, classes=cls_sel, gt_boxes=g(gt["boxes"]), gt_boxes3D=g(gt["boxes3D"]),
                   gt_poses=g(gt["poses"]), fcap=Fcap)
        with torch.no_grad():
            fgm = sel_ok & (cls_sel >= 0) & (cls_sel < K)
            self.stats["roi_head/num_fg_samples"] = fgm.float().sum() / B
            self.stats["roi_head/num_bg_samples"] = (sel_ok & (cls_sel == K)).float().sum() / B
        return out

    # -- pooling + heads ------------------------------------------------------------------------------
    def pool(self, feats, boxes, valid):
        """boxes (B,S,4) -> (B*S, 7*7*C) bf16 NHWC-flattened RoI features (invalid slots pooled from a dummy box)."""
        B, S, _ = boxes.shape
        b = torch.where(valid[:, :, None], boxes, torch.zeros_like(boxes)).reshape(-1, 4)
        bi = torch.arange(B, device=boxes.device, dtype=torch.float32).repeat_interleave(S)
        rois = torch.cat([bi[:, None], assign_levels(b)[:, None], b], 1).contiguous()
        x = ROIAlign.apply(rois, tuple(self.strides), self.pooled, *feats)
        return x.reshape(B * S, -1)

    def box_branch(self, x, split=True, h1=None):
        C, P = self.in_channels, self.pooled
        h = fc(x, self.box_head.fc1, relu=True, chw=(C, P * P)) if h1 is None else h1
        k = 2
        while hasattr(self.box_head, "fc%d" % k):
            h = fc(h, getattr(self.box_head, "fc%d" % k), relu=True)
            k += 1
        n = self.box_predictor.cls_score.weight.shape[0] + self.box_predictor.bbox_pred.weight.shape[0]
        out = fused_predictors(h, [self.box_predictor.cls_score, self.box_predictor.bbox_pred], -(-n // 256) * 256, split)
        return out if not split else (out[0], out[1])

    def box_losses_fused(self, pred, smp):
        """BoxHead losses + logged accuracies from the fused predictor rows in one kernel each way (c3d_box_loss_*)."""
        K = self.num_classes
        o = BoxLoss.apply(pred, smp["classes"].reshape(-1), smp["valid"].reshape(-1), smp["boxes"].reshape(-1, 4),
                          smp["gt_boxes"].reshape(-1, 4), K, self.box_weights)
        with torch.no_grad():
            d = o.detach()
            self.stats["fast_rcnn/cls_accuracy"], self.stats["fast_rcnn/fg_cls_accuracy"] = d[2], d[3]
            self.stats["fast_rcnn/false_negative"] = d[4]
        return {"BoxHead/loss_cls": o[0], "BoxHead/loss_box_reg": o[1]}

    def box_losses(self, scores, deltas, smp):
        K = self.num_classes
        cls = smp["classes"].reshape(-1)
        valid = smp["valid"].reshape(-1)
        n_valid = valid.float().sum().clamp(min=1.0)
        ce = F.cross_entropy(scores, cls.clamp(min=0), reduction="none")
        loss_cls = (ce * valid.float()).sum() / n_valid
        fg = valid & (cls >= 0) & (cls < K)
        d = deltas.view(-1, K, 4)
        pick = torch.gather(d, 1, cls.clamp(0, K - 1)[:, None, None].expand(-1, 1, 4)).squeeze(1)
        tgt = get_deltas(smp["boxes"].reshape(-1, 4), smp["gt_boxes"].reshape(-1, 4), self.box_weights)
        l1 = (pick - tgt).abs().sum(-1)
        loss_box = torch.where(fg, l1, torch.zeros_like(l1)).sum() / n_valid
        with torch.no_grad():
            pred = scores.argmax(1)
            nfg = fg.float().sum().clamp(min=1)
            self.stats["fast_rcnn/cls_accuracy"] = ((pred == cls) & valid).float().sum() / n_valid
            self.stats["fast_rcnn/fg_cls_accuracy"] = ((pred == cls) & fg).float().sum() / nfg
            self.stats["fast_rcnn/false_negative"] = ((pred == K) & fg).float().sum() / nfg
        return {"BoxHead/loss_cls": loss_cls, "BoxHead/loss_box_reg": loss_box}

    def cube_outputs(self, x, classes):
        """x (n, 7*7*C) bf16, classes (n,) -> per-class gathered raw head outputs (fp32)."""
        ch, C, P, K = self.cube_head, self.in_channels, self.pooled, self.num_classes
        fg = ch.feature_generator
        h = fc(x, fg.fc1, relu=True, chw=(C, P * P))
        k = 2
        while hasattr(fg, "fc%d" % k):
            h = fc(h, getattr(fg, "fc%d" % k), relu=True)
            k += 1
        n = x.shape[0]
        c = classes.clamp(0, K - 1)
        heads = [ch.bbox_3D_center_deltas, ch.bbox_3D_dims, ch.bbox_3D_pose, ch.bbox_3D_center_depth, ch.bbox_3D_uncertainty]
        tot = sum(l.weight.shape[0] for l in heads)
        outs = fused_predictors(h, heads, -(-tot // 256) * 256)          # one GEMM for the five K-way predictors
        pick = lambda o, m: torch.gather(o.reshape(n, K, m), 1, c[:, None, None].expand(-1, 1, m)).squeeze(1)
        ur = pick(outs[4], 1).squeeze(1)
        return dict(deltas=pick(outs[0], 2), dims=pick(outs[1], 3), pose6=pick(outs[2], 6),
                    z=pick(outs[3], 1).squeeze(1), uncert=ur.clip(0.01), uncert_raw=ur)

    def cube_pred(self, x, h1=None):
        """x (n, 7*7*C) bf16 -> the five K-way predictors as one fp32 (n, ld) GEMM output [deltas 2K | dims 3K | pose 6K | z K |
        uncertainty K | pad] (cube_head.py:108-144 behind the shared FC stack :63-73)."""
        ch, C, P = self.cube_head, self.in_channels, self.pooled
        fg = ch.feature_generator
        h = fc(x, fg.fc1, relu=True, chw=(C, P * P)) if h1 is None else h1
        k = 2
        while hasattr(fg, "fc%d" % k):
            h = fc(h, getattr(fg, "fc%d" % k), relu=True)
            k += 1
        heads = [ch.bbox_3D_center_deltas, ch.bbox_3D_dims, ch.bbox_3D_pose, ch.bbox_3D_center_depth, ch.bbox_3D_uncertainty]
        tot = sum(l.weight.shape[0] for l in heads)
        return fused_predictors(h, heads, -(-tot // 256) * 256, split=False)

    def cube_losses_kernel(self, pred, boxes, classes, valid, gt3, gtR, meta, per_image):
        """the six Cube losses + logged statistics straight from the fused predictor output: gather / decode + disentangled
        losses / masked finite means = 3 launches each way (CubeHeadLoss), instead of ~330 torch launches."""
        w = self.w
        prior = self.priors_dims_per_cat.detach()[0, :, 0, :]
        o = CubeHeadLoss.apply(pred, classes, valid, boxes, meta, prior, gt3[:, :9], gtR.reshape(-1, 9), per_image,
                               self.num_classes, float(self.virtual_focal))
        w3 = w["w3d"]
        losses = {"Cube/uncert": w["conf"] * o[0], "Cube/loss_dims": o[1] * (w["dims"] * w3), "Cube/loss_xy": o[2] * (w["xy"] * w3),
                  "Cube/loss_z": o[3] * (w["z"] * w3), "Cube/loss_pose": o[4] * (w["pose"] * w3),
                  "Cube/loss_joint": o[5] * (w["joint"] * w3)}
        with torch.no_grad():
            d = o.detach()
            self.stats.update({"Cube/z_error": d[6], "Cube/dims_error": d[7], "Cube/xy_error": d[8], "Cube/z_close": d[9],
                               "Cube/conf": d[10]})
        return losses

    def decode(self, raw, boxes, classes, Kb, v2r):
        """roi_heads.py:409-525: 2D centre, dims (exp * prior), egocentric pose, metric depth."""
        sw, sh = boxes[:, 2] - boxes[:, 0], boxes[:, 3] - boxes[:, 1]
        cx = boxes[:, 0] + 0.5 * sw + sw * raw["deltas"][:, 0]
        cy = boxes[:, 1] + 0.5 * sh + sh * raw["deltas"][:, 1]
        prior = self.priors_dims_per_cat.detach()[0, classes.clamp(0, self.num_classes - 1), 0, :]
        dims = torch.exp(raw["dims"].clip(max=5)) * prior
        pose = G.R_from_allocentric(Kb, G.rotation_6d_to_matrix(raw["pose6"]), cx.detach(), cy.detach())
        return cx, cy, dims, pose, raw["z"] * v2r

    def cube_losses_fused(self, raw, boxes, classes, valid, gt3, gtR, Kb, v2r):
        """same quantities as cube_losses(), computed by the fused sm_90a kernel (c3d_cube_loss_fwd/bwd)."""
        from ..nnfunc import CubeLossRows
        w = self.w
        n = boxes.shape[0]
        prior = self.priors_dims_per_cat.detach()[0, classes.clamp(0, self.num_classes - 1), 0, :]
        aux = torch.cat([boxes, Kb[:, 0, 0:1], Kb[:, 1, 1:2], Kb[:, 0, 2:3], Kb[:, 1, 2:3], v2r[:, None], prior, gt3[:, :6],
                         gtR.reshape(n, 9), boxes.new_zeros(n, 1)], 1)
        raw13 = torch.cat([raw["deltas"], raw["z"][:, None], raw["dims"], raw["pose6"], raw["uncert_raw"][:, None]], 1)
        rows = CubeLossRows.apply(raw13, aux)
        fm = lambda col, m=valid: G.finite_mean(rows[:, col], m)
        losses = {"Cube/uncert": w["conf"] * fm(0), "Cube/loss_dims": fm(1) * w["dims"] * w["w3d"],
                  "Cube/loss_xy": fm(2) * w["xy"] * w["w3d"], "Cube/loss_z": fm(3) * w["z"] * w["w3d"],
                  "Cube/loss_pose": fm(4) * w["pose"] * w["w3d"], "Cube/loss_joint": fm(5) * w["joint"] * w["w3d"]}
        with torch.no_grad():
            r = rows.detach()
            nv = valid.float().sum().clamp(min=1)
            mean = lambda t: torch.where(valid, t, torch.zeros_like(t)).sum() / nv
            self.stats.update({"Cube/z_error": mean(r[:, 6]), "Cube/dims_error": mean(r[:, 7]), "Cube/xy_error": mean(r[:, 8]),
                               "Cube/z_close": mean((r[:, 6] < 0.20).float()), "Cube/conf": mean(r[:, 9])})
        return losses

    def cube_losses(self, raw, boxes, classes, valid, gt3, gtR, Kb, v2r):
        w = self.w
        cx, cy, dims, pose, z = self.decode(raw, boxes, classes, Kb, v2r)
        uncert = raw["uncert"]
        fx, fy, px, py = Kb[:, 0, 0], Kb[:, 1, 1], Kb[:, 0, 2], Kb[:, 1, 2]
        g2, gz, gdims = gt3[:, :2], gt3[:, 2], gt3[:, 3:6]
        lift = lambda zz, uu, vv: torch.stack((zz * (uu - px) / fx, zz * (vv - py) / fy, zz), 1)
        g3 = lift(gz, g2[:, 0], g2[:, 1])
        gt_c = G.cuboid_corners(g3, gdims, gtR)
        n = boxes.shape[0]
        l1 = lambda c: (c - gt_c).abs().reshape(n, -1).mean(1)
        loss_z = l1(G.cuboid_corners(lift(z, g2[:, 0], g2[:, 1]), gdims, gtR))
        loss_xy = l1(G.cuboid_corners(lift(gz, cx, cy), gdims, gtR))
        loss_dims = l1(G.cuboid_corners(g3, dims, gtR))
        loss_pose = G.chamfer8(G.cuboid_corners(g3, gdims, pose), gt_c)
        loss_joint = G.chamfer8(G.cuboid_corners(lift(z, cx, cy), dims, pose), gt_c)
        sf = SQRT2 * torch.exp(-uncert)
        fm = lambda l, m=valid: G.finite_mean(l, m)
        losses = {"Cube/uncert": w["conf"] * fm(uncert),
                  "Cube/loss_dims": fm(loss_dims * sf) * w["dims"] * w["w3d"],
                  "Cube/loss_xy": fm(loss_xy * sf) * w["xy"] * w["w3d"],
                  "Cube/loss_z": fm(loss_z * sf) * w["z"] * w["w3d"],
                  "Cube/loss_pose": fm(loss_pose * sf) * w["pose"] * w["w3d"],
                  "Cube/loss_joint": fm(loss_joint * sf, valid & (loss_joint < float("inf"))) * w["joint"] * w["w3d"]}
        with torch.no_grad():
            vm = valid.float()
            nv = vm.sum().clamp(min=1)
            mean = lambda t: (torch.where(valid, t, torch.zeros_like(t))).sum() / nv
            z_err = (z - gz).abs()
            total = loss_dims * w["dims"] + loss_pose * w["pose"] + loss_xy * w["xy"] + loss_z * w["z"] + loss_joint * w["joint"]
            self.stats.update({"Cube/z_error": mean(z_err), "Cube/dims_error": mean((dims - gdims).abs().mean(1)),
                               "Cube/xy_error": mean((torch.stack((cx, cy), 1) - g2).abs().mean(1)),
                               "Cube/z_close": mean((z_err < 0.20).float()),
                               "Cube/total_3D_loss": w["w3d"] * fm(total), "Cube/conf": mean(torch.exp(-uncert))})
        return losses

    def per_box_camera(self, Ks, ratios, im_h, counts_or_S, B, device):
        """scaled intrinsics per box and the virtual->real depth factor (roi_heads.py:372-404)."""
        if torch.is_tensor(Ks):
            K = Ks
        else:
            K = torch.stack([torch.as_tensor(k, dtype=torch.float32) for k in Ks]).to(device)     # (B,3,3)
        r = ratios if torch.is_tensor(ratios) else torch.as_tensor(ratios, dtype=torch.float32, device=device)
        Ks_scaled = K / r[:, None, None]
        Ks_scaled[:, 2, 2] = 1
        h = im_h if torch.is_tensor(im_h) else torch.as_tensor(im_h, dtype=torch.float32, device=device)
        v2r = (h * K[:, 1, 1]) / (self.virtual_focal * (h * r))
        rep = lambda t: t.repeat_interleave(counts_or_S, dim=0)
        return rep(Ks_scaled), rep(v2r), rep(r)

    # -- forward ----------------------------------------------------------------------------------------
    def forward(self, features, proposals, image_sizes, Ks, ratios, gt=None, im_h=None, meta=None):
        feats = [features[f] for f in self.in_features]
        prop_boxes, prop_scores, prop_count = proposals
        B = prop_boxes.shape[0]
        dev = prop_boxes.device
        if im_h is None:
            im_h = [s[0] for s in image_sizes]
        if self.training:
            smp = self.label_and_sample_proposals(prop_boxes, prop_count, gt)
            x = self.pool(feats, smp["boxes"], smp["valid"])
            fused = self.fused_head_losses and meta is not None and self.fused_cube and x.is_cuda
            Fc = min(smp["fcap"], smp["boxes"].shape[1])
            hb1 = hc1 = None
            if fused and self.share_pool and x.shape[0] == B * smp["boxes"].shape[1]:
                # both heads' first FC layer on the ONE pooled tensor (the cube head's RoIs are rows [:Fc] of every image)
                hb1, hc1 = TwoHeadFC1.apply(x, self.box_head.fc1.weight, self.box_head.fc1.bias,
                                            self.cube_head.feature_generator.fc1.weight, self.cube_head.feature_generator.fc1.bias,
                                            B, smp["boxes"].shape[1], Fc, (self.in_channels, self.pooled * self.pooled))
            if fused:
                losses = self.box_losses_fused(self.box_branch(x, split=False, h1=hb1), smp)
            else:
                scores, deltas = self.box_branch(x)
                losses = self.box_losses(scores, deltas, smp)
            K = self.num_classes
            fb, fc_, fv = smp["boxes"][:, :Fc], smp["classes"][:, :Fc], smp["valid"][:, :Fc]
            fv = fv & (fc_ >= 0) & (fc_ < K)
            if hc1 is not None:
                xc = None
            elif self.share_pool:
                xc = x.view(B, -1, x.shape[-1])[:, :Fc].reshape(B * Fc, -1)
            else:
                xc = self.pool(feats, fb, fv)
            if fused:
                losses.update(self.cube_losses_kernel(self.cube_pred(xc, h1=hc1), fb.reshape(-1, 4), fc_.reshape(-1), fv.reshape(-1),
                                                      smp["gt_boxes3D"][:, :Fc].reshape(-1, 9),
                                                      smp["gt_poses"][:, :Fc].reshape(-1, 3, 3), meta, Fc))
                return None, losses
            Kb, v2r, _ = self.per_box_camera(Ks, ratios, im_h, Fc, B, dev)
            raw = self.cube_outputs(xc, fc_.reshape(-1))
            cube_fn = self.cube_losses_fused if self.fused_cube else self.cube_losses
            losses.update(cube_fn(raw, fb.reshape(-1, 4), fc_.reshape(-1), fv.reshape(-1),
                                           smp["gt_boxes3D"][:, :Fc].reshape(-1, 9), smp["gt_poses"][:, :Fc].reshape(-1, 3, 3),
                                           Kb, v2r))
            return None, losses
        return self.inference(feats, prop_boxes, prop_count, image_sizes, Ks, ratios), {}

    # -- inference (fast_rcnn.py:57-143 + roi_heads.py:227-246,774-819), batched over all images ---------------
    @torch.no_grad()
    def box_dense(self, feats, prop_boxes, prop_count):
        """-> probs (B,P,K+1) softmax scores, boxes (B,P,K,4) per-class decoded boxes (FastRCNNOutputLayers.predict_*)."""
        B, P, _ = prop_boxes.shape
        K = self.num_classes
        pvalid = torch.arange(P, device=prop_boxes.device)[None] < prop_count[:, None]
        x = self.pool(feats, prop_boxes, pvalid)
        scores, deltas = self.box_branch(x)
        probs = F.softmax(scores, -1).view(B, P, K + 1)
        pboxes = apply_deltas(deltas.contiguous(), prop_boxes.reshape(-1, 4), self.box_weights).view(B, P, K, 4)
        return probs, pboxes

    @torch.no_grad()
    def select_detections(self, probs, pboxes, prop_count, hw, max_candidates=8192):
        """fast_rcnn_inference for ALL images without a per-image loop (SURVEY 8f-2): finite / score filter + clip
        (c3d_det_candidates) -> top-M candidates in score order (c3d_topk_segments) -> per-class greedy NMS
        (c3d_nms_batched, categories = classes) -> first DETECTIONS_PER_IMAGE survivors.
        -> boxes (B,D,4), scores (B,D), classes (B,D), scores_full (B,D,K), proposal index (B,D), count (B,) — identical to
        the per-image reference whenever the D-th survivor lies inside the top-M candidates (checked; else exact rounds)."""
        from .. import kernels as Kx
        B, P, K1 = probs.shape
        K, D = K1 - 1, self.test_topk
        cs, cb, maxc, total = Kx.det_candidates(probs, pboxes, prop_count, hw, self.test_score_thresh)
        M = min(P * K, max_candidates)
        sv, si, cnt = Kx.topk_segments([(cs, M)], want_idx64=True, want_counts=True)
        sb = torch.gather(cb, 1, si[:, :, None].expand(-1, -1, 4))
        cats = (si % K).float()
        keep, kcnt = Kx.nms_batched(sb, cnt.reshape(-1).contiguous(), self.test_nms_thresh, D, cats=cats, maxc=maxc,
                                    trick_max_numel=self.nms_trick_max_numel)
        safe = keep.clamp(min=0).long()
        flat = torch.gather(si, 1, safe)
        out = dict(boxes=torch.gather(sb, 1, safe[:, :, None].expand(-1, -1, 4)), scores=torch.gather(sv, 1, safe),
                   classes=flat % K, prop=flat // K, count=kcnt)
        host = torch.stack([kcnt, total]).tolist()            # the ONE device->host read of the post-processing
        for i in range(B):
            if host[0][i] < D and host[1][i] > M:             # the D-th survivor may lie beyond the top-M: exact rounds
                self._select_rounds(i, cs, cb, maxc, out, M, D, K)
                host[0][i] = int(out["count"][i])
        out["scores_full"] = torch.gather(probs[:, :, :K], 1, out["prop"][:, :, None].expand(-1, -1, K))
        out["counts_host"] = host[0]
        return out

    @torch.no_grad()
    def _select_rounds(self, i, cs, cb, maxc, out, M, D, K):
        """rare path of select_detections for one image: walk the fully sorted candidate list in chunks, every chunk
        preceded by the survivors so far (they are higher-scored and mutually compatible, so the greedy scan keeps them)."""
        from .. import kernels as Kx
        score, order = cs[i].sort(descending=True)
        n = int(torch.isfinite(score).sum())
        kept = torch.zeros(0, dtype=torch.long, device=cs.device)        # indices into the candidate array
        pos = 0
        while pos < n and kept.numel() < D:
            chunk = order[pos:min(n, pos + M - kept.numel())]
            idx = torch.cat([kept, chunk])
            pos += chunk.numel()
            nv = torch.tensor([idx.numel()], dtype=torch.int32, device=cs.device)
            keep, kc = Kx.nms_batched(cb[i][idx][None].contiguous(), nv, self.test_nms_thresh, D, cats=(idx % K).float()[None],
                                      maxc=maxc[i:i + 1], trick_max_numel=0)
            kept = idx[keep[0, :int(kc[0])].long()]
        c = kept.numel()
        out["boxes"][i, :c], out["scores"][i, :c] = cb[i][kept], cs[i][kept]
        out["classes"][i, :c], out["prop"][i, :c], out["count"][i] = kept % K, kept // K, c

    @torch.no_grad()
    def cube_decode(self, feats, boxes, classes, valid, image_sizes, Ks, ratios):
        """roi_heads.py:326-524,774-819 at inference for (B,D) detections -> dict of (B*D, ...) 3D outputs."""
        B, D, _ = boxes.shape
        dev = boxes.device
        xc = self.pool(feats, boxes, valid)
        Kb, v2r, rr = self.per_box_camera(Ks, ratios, [s[0] for s in image_sizes], D, B, dev)
        raw = self.cube_outputs(xc, classes.reshape(-1))
        cx, cy, dims, pose, z = self.decode(raw, boxes.reshape(-1, 4), classes.reshape(-1), Kb, v2r)
        fx, fy, px, py = Kb[:, 0, 0], Kb[:, 1, 1], Kb[:, 0, 2], Kb[:, 1, 2]
        cam = torch.stack((z * (cx - px) / fx, z * (cy - py) / fy, z), 1)
        return dict(cam=cam, dims=dims, pose=pose, conf=torch.exp(-raw["uncert"]), c2d=torch.stack((cx, cy), 1) * rr[:, None],
                    corners=G.cuboid_corners(cam, dims, pose))

    @torch.no_grad()
    def inference(self, feats, prop_boxes, prop_count, image_sizes, Ks, ratios, hw=None):
        from .structures import Boxes, Instances
        B = prop_boxes.shape[0]
        dev = prop_boxes.device
        if hw is None:
            hw = torch.as_tensor(image_sizes, dtype=torch.float32, device=dev)
        probs, pboxes = self.box_dense(feats, prop_boxes, prop_count)
        det = self.select_detections(probs, pboxes, prop_count, hw)
        D = det["boxes"].shape[1]
        valid = torch.arange(D, device=dev)[None] < det["count"][:, None]
        c3 = self.cube_decode(feats, det["boxes"], det["classes"], valid, image_sizes, Ks, ratios)
        scores = (det["scores"].reshape(-1) * c3["conf"]) ** 0.5
        results = []
        for i, n in enumerate(det["counts_host"]):               # views only: no device work, no host sync
            sl = slice(i * D, i * D + n)
            inst = Instances(tuple(image_sizes[i]))
            inst.pred_boxes = Boxes(det["boxes"][i, :n]); inst.scores = scores[sl]
            inst.scores_full = det["scores_full"][i, :n]; inst.pred_classes = det["classes"][i, :n]
            inst.pred_bbox3D = c3["corners"][sl]; inst.pred_center_cam = c3["cam"][sl]; inst.pred_center_2D = c3["c2d"][sl]
            inst.pred_dimensions = c3["dims"][sl]; inst.pred_pose = c3["pose"][sl]
            results.append(inst)
        return results
