"""RCNN3D meta-architecture + build_model on the accelerated path
(cubercnn/modeling/meta_arch/rcnn3d.py:25-112, 247-272).

Call signature of the reference: model(batched_inputs: List[Dict]) -> training: dict of the 10 loss tensors
(rcnn3d.py:74-77); eval: list of {"instances": Instances}.  Input dicts carry `image` (3,H,W) BGR,
`height`, `width`, `K` and in training either `instances` (an object exposing gt_classes, gt_boxes(.tensor),
gt_boxes3D, gt_poses — cubercnn/data/dataset_mapper.py:133-155) or the plain `gt` dict of
omni3d_b200.synth.  EventStorage scalars the reference logs with .item() syncs are kept as device tensors
in `model.metrics` (one async read by the caller instead of ~20 host syncs per step).
"""
import torch
from torch import nn

from .. import _lib
from .. import kernels as Kx
from ..nnfunc import fork
from .backbone import FPN  # noqa: F401  (registers the builders)
from .registry import BACKBONE_REGISTRY, META_ARCH_REGISTRY, PROPOSAL_GENERATOR_REGISTRY, ROI_HEADS_REGISTRY
from .roi_heads import ROIHeads3D  # noqa: F401
from .rpn import RPNWithIgnore  # noqa: F401
from .structures import Boxes, Instances


def _gt_fields(item):
    if "gt" in item:
        g = item["gt"]
        return g["classes"], g["boxes"], g["boxes3D"], g["poses"]
    inst = item["instances"]
    boxes = inst.gt_boxes.tensor if hasattr(inst.gt_boxes, "tensor") else inst.gt_boxes
    return inst.gt_classes, boxes, inst.gt_boxes3D, inst.gt_poses


def collate_gt(batched_inputs, device):
    """list of per-image GT -> padded (B,G,...) tensors + `present` mask (one H2D copy per field)."""
    fields = [_gt_fields(it) for it in batched_inputs]
    B, Gm = len(fields), max(max(len(f[0]) for f in fields), 1)
    src = fields[0][0].device                      # build where the annotations live (host, or HBM-resident)
    if all(len(f[0]) == Gm for f in fields):       # equal counts (synthetic / bucketed batches): 5 stacks instead of 5*B slice copies
        mv = lambda t: t.to(device, non_blocking=True)
        return {"classes": mv(torch.stack([f[0] for f in fields]).long()), "boxes": mv(torch.stack([f[1] for f in fields]).float()),
                "boxes3D": mv(torch.stack([f[2][:, :9] for f in fields]).float()),
                "poses": mv(torch.stack([f[3] for f in fields]).float()),
                "present": mv(torch.ones((B, Gm), dtype=torch.bool, device=src))}
    cls = torch.full((B, Gm), -2, dtype=torch.long, device=src)
    boxes = torch.zeros((B, Gm, 4), device=src)
    b3d = torch.zeros((B, Gm, 9), device=src)
    poses = torch.eye(3, device=src).repeat(B, Gm, 1, 1)
    present = torch.zeros((B, Gm), dtype=torch.bool, device=src)
    for i, (c, b, b3, p) in enumerate(fields):
        n = len(c)
        cls[i, :n], boxes[i, :n], b3d[i, :n], poses[i, :n], present[i, :n] = c, b, b3[:, :9], p, True
    mv = lambda t: t.to(device, non_blocking=True)
    return {"classes": mv(cls), "boxes": mv(boxes), "boxes3D": mv(b3d), "poses": mv(poses), "present": mv(present)}


@META_ARCH_REGISTRY.register()
class RCNN3D(nn.Module):
    def __init__(self, cfg, priors=None):
        super().__init__()
        _lib.lib()       # fail loudly when libc3d.so is missing: there is no CPU / library fallback
        self.backbone = BACKBONE_REGISTRY.get(cfg.MODEL.BACKBONE.NAME)(cfg, None, priors)
        strides, ch = self.backbone.out_strides, self.backbone.out_channels
        self.proposal_generator = PROPOSAL_GENERATOR_REGISTRY.get(cfg.MODEL.PROPOSAL_GENERATOR.NAME)(cfg, ch, strides)
        self.roi_heads = ROI_HEADS_REGISTRY.get(cfg.MODEL.ROI_HEADS.NAME)(cfg, ch, strides, priors=priors)
        self.register_buffer("pixel_mean", torch.tensor(cfg.MODEL.PIXEL_MEAN).view(-1, 1, 1), False)
        self.register_buffer("pixel_std", torch.tensor(cfg.MODEL.PIXEL_STD).view(-1, 1, 1), False)
        self._mean = [float(v) for v in cfg.MODEL.PIXEL_MEAN]
        self._std = [float(v) for v in cfg.MODEL.PIXEL_STD]
        self.input_format = cfg.INPUT.FORMAT
        self.vis_period = cfg.VIS_PERIOD
        self.metrics = {}

    @property
    def device(self):
        return self.pixel_mean.device

    late_parameter_prefix = "backbone.bottom_up."

    def set_backward_cut(self, enable):
        """FlatSGDTrainer (several ranks): cut the autograd graph at the bottom-up backbone's outputs so that
        loss.backward() ends above the backbone and `backward_cut()` hands over the feature gradients for stage 2.
        Never enable this without a trainer that runs stage 2 — the backbone would receive no gradient."""
        self.backbone.split_backward = bool(enable)

    def backward_cut(self):
        """-> (bottom-up outputs, their gradients from stage 1) of the last forward, or None when the graph was not cut."""
        cut = getattr(self.backbone, "cut", None)
        if not cut:
            return None
        src, leaves = cut
        self.backbone.cut = None
        keys = [k for k in src if leaves[k].grad is not None]
        return [src[k] for k in keys], [leaves[k].grad for k in keys]

    def preprocess_image(self, batched_inputs):
        st = self.stage_inputs(batched_inputs, with_gt=False)
        return self._normalize(st), st["sizes"]

    def _normalize(self, st):
        return Kx.preprocess_images(st["images"], self._mean, self._std, self.backbone.size_divisibility,
                                    cpad=getattr(self.backbone.bottom_up, "stem_cpad", 16))

    def stage_inputs(self, batched_inputs, with_gt=True):
        """ALL host->device traffic of a step, and nothing else: images (uint8 as the mapper emits them, or float),
        one (B,12) row of per-image scalars [h, w, height/h, K (9)], and the padded GT.  `forward_staged` consumes
        only these device tensors (no host reads), so it can be recorded into a CUDA graph."""
        dev = self.device
        imgs = [x["image"].to(dev, non_blocking=True) for x in batched_inputs]
        imgs = [(im if im.dtype == torch.uint8 else im.float()).contiguous() for im in imgs]
        sizes = [(int(im.shape[1]), int(im.shape[2])) for im in imgs]
        rows = [[float(h), float(w), info["height"] / h] + [float(v) for r in info["K"] for v in r]
                for info, (h, w) in zip(batched_inputs, sizes)]
        meta = torch.tensor(rows, dtype=torch.float32)
        if dev.type == "cuda":
            meta = meta.pin_memory()
        st = {"images": imgs, "sizes": sizes, "meta": meta.to(dev, non_blocking=True)}
        if with_gt and self.training:
            st["gt"] = collate_gt(batched_inputs, dev)
        return st

    def forward_staged(self, st, _inject=None, batched_inputs=None):
        x = self._normalize(st)
        sizes, meta = st["sizes"], st["meta"]
        hw, ratios, Ks = meta[:, :2], meta[:, 2], meta[:, 3:12].reshape(-1, 3, 3)
        if self.training:
            gt = dict(st["gt"])
            if _inject:
                gt.update(_inject)
            features = self.backbone(x)
            # every FPN map feeds the RPN head AND the RoI pooler: one alias per consumer, so the RPN conv's data gradient
            # is added into the pooler's gradient inside the conv epilogue (nnfunc.fork) instead of by an add pass
            f_rpn, f_roi = {}, {}
            for k, v in features.items():
                f_rpn[k], f_roi[k] = fork(v, 2)
            proposals, l_rpn = self.proposal_generator(f_rpn, sizes, gt, sizes_dev=hw)
            _, losses = self.roi_heads(f_roi, proposals, sizes, Ks, ratios, gt, im_h=hw[:, 0], meta=meta)
            losses.update(l_rpn)
            self.metrics = {**self.proposal_generator.stats, **self.roi_heads.stats}
            return losses
        features = self.backbone(x)
        proposals, _ = self.proposal_generator(features, sizes, None, sizes_dev=hw)
        results, _ = self.roi_heads(features, proposals, sizes, Ks, ratios, None, im_h=hw[:, 0])
        return self._postprocess(results, batched_inputs, sizes)

    def forward(self, batched_inputs, _inject=None):
        if self.device.type != "cuda":
            raise _lib.C3DError("omni3d_b200 RCNN3D runs on CUDA only (MODEL.DEVICE=cpu is the oracle's job)")
        return self.forward_staged(self.stage_inputs(batched_inputs), _inject, batched_inputs)

    inference = forward

    @staticmethod
    def _postprocess(results, batched_inputs, sizes):
        out = []
        for r, inp, (h, w) in zip(results, batched_inputs, sizes):
            oh, ow = inp.get("height", h), inp.get("width", w)
            sx, sy = ow / w, oh / h
            b = r.pred_boxes.tensor.clone()
            b[:, 0::2] = (b[:, 0::2] * sx).clamp(0, ow)
            b[:, 1::2] = (b[:, 1::2] * sy).clamp(0, oh)
            keep = ((b[:, 2] - b[:, 0]) > 0) & ((b[:, 3] - b[:, 1]) > 0)
            new = Instances((int(oh), int(ow)), **{k: v for k, v in r.get_fields().items() if k != "pred_boxes"})
            new.pred_boxes = Boxes(b)
            out.append({"instances": new[keep]})
        return out


def build_model(cfg, priors=None):
    """rcnn3d.py:247-256."""
    model = META_ARCH_REGISTRY.get(cfg.MODEL.META_ARCHITECTURE)(cfg, priors=priors)
    model.to(torch.device(cfg.MODEL.DEVICE))
    return model
