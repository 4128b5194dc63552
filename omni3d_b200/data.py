"""Device-side input pipeline — SURVEY 8f-3.

Mirror of cubercnn/data/dataset_mapper.py:17-155 (DatasetMapper3D.__call__, transform_instance_annotations,
annotations_to_instances) with the reference's train-time augmentations (detectron2 defaults selected by
configs/Base.yaml:10-13 + config.py:147: T.ResizeShortestEdge(MIN_SIZE_TRAIN, MAX_SIZE_TRAIN, "choice") and
T.RandomFlip(horizontal)) re-designed for the GPU: the decoded uint8 image goes to the GPU ONCE, as it is; resize
(Pillow-exact 8-bit bilinear, what detectron2's ResizeTransform calls), flip and the HWC->CHW transposition run there
(c3d_resize_bilinear_u8) and hand the model the same uint8 (3,H,W) tensor the reference's mapper emits — no CPU resample,
no deepcopy, no per-image pickle through worker queues.  The few annotation numbers are transformed on the host in float64
exactly like the reference and collated into the padded device tensors RCNN3D.stage_inputs consumes.

    resize_flip_u8(img_hwc_u8, new_h, new_w, flip)         -> (3,new_h,new_w) uint8 CUDA tensor (== Pillow, bit for bit)
    shortest_edge_shape(h, w, size, max_size)               -> (new_h, new_w)   (ResizeShortestEdge.get_output_shape)
    DeviceMapper3D(cfg, is_train)(record[, size, flip])     -> {"image", "height", "width", "K", "gt"}
"""
import math

import numpy as np
import torch

from . import _lib

PRECISION_BITS = 32 - 8 - 2
_coef_cache = {}


def pil_bilinear_coeffs(in_size, out_size):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc for the triangle filter over a whole axis (vectorised; the
    scalar restatement pinned against Pillow lives in oracle/pil_resize.py): -> bounds (out,2) int32 [first, count],
    kk (out, ksize) int32 weights in 22-bit fixed point."""
    scale = float(np.float32(np.float32(in_size) - np.float32(0.0))) / out_size
    fs = max(scale, 1.0)
    support = fs
    ksize = int(math.ceil(support)) * 2 + 1
    xx = np.arange(out_size, dtype=np.float64)
    center = 0.0 + (xx + 0.5) * scale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)          # C cast: truncation of a positive value
    xmin = np.where(center - support + 0.5 < 0, 0, xmin)
    xmax = np.minimum((center + support + 0.5).astype(np.int64), in_size)
    cnt = xmax - xmin
    x = np.arange(ksize, dtype=np.float64)[None, :]
    a = np.abs((x + xmin[:, None] - center[:, None] + 0.5) * (1.0 / fs))
    w = np.where(a < 1.0, 1.0 - a, 0.0)
    w = np.where(x < cnt[:, None], w, 0.0)
    # sequential left-to-right sum like the C loop (ww += w) — np.cumsum accumulates in the same order
    ww = np.cumsum(w, axis=1)[:, -1:]
    w = np.where(ww != 0.0, w / np.where(ww != 0.0, ww, 1.0), w)
    kk = (0.5 + w * float(1 << PRECISION_BITS)).astype(np.int64).astype(np.int32)            # weights are >= 0
    return np.stack([xmin, cnt], 1).astype(np.int32), np.ascontiguousarray(kk)


def _coeffs_dev(in_size, out_size, device):
    key = (in_size, out_size, device.index)
    hit = _coef_cache.get(key)
    if hit is None:
        b, k = pil_bilinear_coeffs(in_size, out_size)
        hit = (torch.from_numpy(b).to(device), torch.from_numpy(k).to(device), k.shape[1], int(b[0, 0]), int(b[-1, 0] + b[-1, 1]))
        if len(_coef_cache) > 512:
            _coef_cache.clear()
        _coef_cache[key] = hit
    return hit


def shortest_edge_shape(h, w, size, max_size):
    """detectron2 ResizeShortestEdge.get_output_shape."""
    scale = size * 1.0 / min(h, w)
    if h < w:
        newh, neww = size, scale * w
    else:
        newh, neww = scale * h, size
    if max(newh, neww) > max_size:
        scale = max_size * 1.0 / max(newh, neww)
        newh, neww = newh * scale, neww * scale
    return int(newh + 0.5), int(neww + 0.5)


def resize_flip_u8(img, new_h, new_w, flip=False):
    """img (H,W,3) uint8 (CUDA tensor, or host tensor / array: copied once) -> (3,new_h,new_w) uint8 CUDA tensor equal to
    np.asarray(Image.fromarray(img).resize((new_w,new_h), BILINEAR))[:, ::-1 if flip].transpose(2,0,1)."""
    L = _lib.lib()
    if not torch.cuda.is_available():
        raise _lib.C3DError("omni3d_b200.data needs a CUDA device (no CPU fallback)")
    if not isinstance(img, torch.Tensor):
        img = torch.from_numpy(np.ascontiguousarray(img))
    if not img.is_cuda:
        img = img.pin_memory().cuda(non_blocking=True)
    assert img.dtype == torch.uint8 and img.dim() == 3
    img = img.contiguous()
    H, W, C = img.shape
    dev = img.device
    bh, kh, ksh, _, _ = _coeffs_dev(W, new_w, dev)
    bv, kv, ksv, first, last = _coeffs_dev(H, new_h, dev)
    tmp = torch.empty((H, new_w, C), dtype=torch.uint8, device=dev)
    out = torch.empty((C, new_h, new_w), dtype=torch.uint8, device=dev)
    _lib.check(L.c3d_resize_bilinear_u8(img.data_ptr(), H, W, C, bh.data_ptr(), kh.data_ptr(), ksh, bv.data_ptr(), kv.data_ptr(), ksv,
                                        new_h, new_w, first, last, int(bool(flip)), tmp.data_ptr(), out.data_ptr(),
                                        _lib.stream(dev)), launches=2)
    return out


_M1 = np.array([[1.0, 0, 0], [0, -1, 0], [0, 0, -1]])
_M2 = np.array([[-1.0, 0, 0], [0, -1, 0], [0, 0, 1]])


def transform_annotations(annos, K, h, w, new_h, new_w, flip):
    """transform_instance_annotations + annotations_to_instances (dataset_mapper.py:74-155) for all objects of an image at
    once, float64 like the reference: 2D boxes (XYXY_ABS), projected 3D centre, pose mirror.  `annos`: list of the dataset's
    annotation dicts (bbox XYXY abs, center_cam, dimensions, pose, category_id, iscrowd).
    -> {"classes" int64 (n,), "boxes" (n,4), "boxes3D" (n,9) = [u,v,z,W,H,L,X,Y,Z], "poses" (n,3,3)} fp32 tensors."""
    annos = [a for a in annos if a.get("iscrowd", 0) == 0]
    n = len(annos)
    K = np.asarray(K, np.float64)
    sx, sy = new_w * 1.0 / w, new_h * 1.0 / h
    box = np.array([a["bbox"] for a in annos], np.float64).reshape(n, 4)
    box = box * np.array([sx, sy, sx, sy])
    if flip:
        box = np.stack([new_w - box[:, 2], box[:, 1], new_w - box[:, 0], box[:, 3]], 1)
    c3 = np.array([a["center_cam"] for a in annos], np.float64).reshape(n, 3)
    p = (K @ c3.T).T
    nz = c3[:, 2] != 0
    # objects with z == 0 keep the dataset's stored projection untouched (the reference skips them, :86)
    stored = np.array([list(a.get("center_cam_proj", [0.0, 0.0, 0.0]))[:3] for a in annos], np.float64).reshape(n, 3)
    uv = np.zeros((n, 2))
    uv[nz] = p[nz, :2] / p[nz, 2:3]
    uv = uv * np.array([sx, sy])
    if flip:
        uv[:, 0] = new_w - uv[:, 0]
    uv[~nz] = stored[~nz, :2]
    p[~nz, 2] = stored[~nz, 2]
    pose = np.array([a["pose"] for a in annos], np.float64).reshape(n, 3, 3)
    if flip:
        pose = np.where(nz[:, None, None], _M1 @ pose @ _M2, pose)
    dims = np.array([a["dimensions"] for a in annos], np.float64).reshape(n, 3)
    b3 = np.concatenate([uv, p[:, 2:3], dims, c3], 1)
    keep = ((box[:, 2] - box[:, 0]) > 1e-5) & ((box[:, 3] - box[:, 1]) > 1e-5)       # detection_utils.filter_empty_instances
    f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a[keep])).float()
    return {"classes": torch.tensor([int(a["category_id"]) for a, k in zip(annos, keep) if k], dtype=torch.int64),
            "boxes": f32(box), "boxes3D": f32(b3), "poses": f32(pose)}


class DeviceMapper3D:
    """DatasetMapper3D for an already decoded image: record = {"image_hwc": (H,W,3) uint8 BGR array / tensor, "height",
    "width", "K", "annotations": [...]} -> the batched-input dict of RCNN3D (image (3,h',w') uint8 on the GPU, original
    height/width, K, and — in training — the transformed ground truth as plain tensors)."""

    def __init__(self, cfg, is_train=True, seed=None):
        I = cfg.INPUT
        self.is_train = is_train
        self.min_sizes = tuple(I.MIN_SIZE_TRAIN) if is_train else (I.MIN_SIZE_TEST,)
        self.max_size = I.MAX_SIZE_TRAIN if is_train else I.MAX_SIZE_TEST
        self.sampling = I.MIN_SIZE_TRAIN_SAMPLING if is_train else "choice"
        if self.sampling != "choice":
            raise NotImplementedError("INPUT.MIN_SIZE_TRAIN_SAMPLING other than 'choice' (Base.yaml uses 'choice')")
        self.flip = is_train and I.RANDOM_FLIP == "horizontal"
        if is_train and I.RANDOM_FLIP not in ("horizontal", "none"):
            raise NotImplementedError("INPUT.RANDOM_FLIP = %s" % I.RANDOM_FLIP)
        self.rng = np.random.default_rng(seed)

    def __call__(self, record, size=None, flip=None):
        img = record["image_hwc"]
        h, w = int(img.shape[0]), int(img.shape[1])
        if size is None:
            size = int(self.rng.choice(self.min_sizes))
        if flip is None:
            flip = bool(self.flip and self.rng.random() < 0.5)
        new_h, new_w = shortest_edge_shape(h, w, size, self.max_size) if size > 0 else (h, w)
        out = {"image": resize_flip_u8(img, new_h, new_w, flip), "height": record.get("height", h),
               "width": record.get("width", w), "K": record["K"]}
        if self.is_train and "annotations" in record:
            out["gt"] = transform_annotations(record["annotations"], record["K"], h, w, new_h, new_w, flip)
        return out
