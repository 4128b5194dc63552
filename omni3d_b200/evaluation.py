"""Batched 3D-IoU front-end for the evaluator — SURVEY 8f-1.

The reference's only caller of box3d_overlap is Omni3Deval.computeIoU
(cubercnn/evaluation/omni3d_evaluation.py:1359-1431), evaluated once per (image, category) from the dict
comprehension at :1339-1343: tens of thousands of calls with N <= maxDets detections x M <= ~30 ground truths,
each doing two host->device copies, one tiny op and one device->host copy (or, with MAX_DTS_CROSS_GTS_FOR_IOU3D = 0
at :62, a serial CPU loop).  Here ALL (image, category) groups go through ONE segmented launch
(c3d_box3d_overlap_segmented: CSR offsets over the groups, one H2D of the boxes, one D2H of the packed IoUs).

    compute_ious_3d(dts, gts, img_ids, cat_ids, max_dets)  ->  {(imgId, catId): ious}   == self.ious of the reference
    box3d_overlap_segmented(dt_groups, gt_groups)          ->  list of (n_i, m_i) IoU matrices

Semantics kept from the reference: detections sorted by -score with a stable (merge) sort, truncated to maxDets[-1];
`[]` when a group has no detections and no ground truths, or when either side is empty (:1414-1415); dt rows that fail the
planarity / non-zero-volume checks are zeroed and counted in the printed warning (:158-164), once for the whole batch.
"""
import numpy as np
import torch

from . import _lib
from .box3d import _device_of, _workspace

def _as_boxes(x):
    a = np.asarray(x, dtype=np.float32)
    if a.size == 0:
        return np.zeros((0, 8, 3), np.float32)
    if a.ndim != 3 or a.shape[1:] != (8, 3):
        raise ValueError(f"boxes must be (n, 8, 3), got {a.shape}")
    return a


def box3d_overlap_segmented(dt_groups, gt_groups, eps_coplanar=1e-4, eps_nonzero=1e-8, device=None, return_bad_counts=False):
    """dt_groups[i] (n_i,8,3), gt_groups[i] (m_i,8,3) (arrays / tensors / nested lists) -> [iou_i (n_i, m_i) float32 numpy].
    One launch for all groups; equals box3d_overlap(dt_i, gt_i) of every group bit for bit."""
    if len(dt_groups) != len(gt_groups):
        raise ValueError("dt_groups and gt_groups must have the same length")
    L = _lib.lib()
    G = len(dt_groups)
    dts = [_as_boxes(d.cpu() if isinstance(d, torch.Tensor) else d) for d in dt_groups]
    gts = [_as_boxes(g.cpu() if isinstance(g, torch.Tensor) else g) for g in gt_groups]
    nd = np.array([len(d) for d in dts], np.int64)
    ng = np.array([len(g) for g in gts], np.int64)
    dt_off = np.zeros(G + 1, np.int32); dt_off[1:] = np.cumsum(nd)
    gt_off = np.zeros(G + 1, np.int32); gt_off[1:] = np.cumsum(ng)
    pair_off = np.zeros(G + 1, np.int64); pair_off[1:] = np.cumsum(nd * ng)
    n_dt, n_gt, total = int(dt_off[-1]), int(gt_off[-1]), int(pair_off[-1])
    bad = [0, 0]
    out = np.zeros(total, np.float32)
    if n_dt > 0:
        dev = device if device is not None else _device_of()
        with torch.cuda.device(dev):
            up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=False)
            b1 = up(np.concatenate(dts) if n_dt else np.zeros((0, 8, 3), np.float32))
            b2 = up(np.concatenate(gts) if n_gt else np.zeros((1, 8, 3), np.float32))
            d_off, g_off, p_off = up(dt_off), up(gt_off), up(pair_off)
            iou = torch.empty(max(total, 1), dtype=torch.float32, device=dev)
            nbad = torch.zeros(2, dtype=torch.int32, device=dev)
            ws = _workspace(L.c3d_box3d_overlap_segmented_workspace_bytes(n_dt, max(n_gt, 1), total), dev)
            _lib.check(L.c3d_box3d_overlap_segmented(b1.data_ptr(), n_dt, b2.data_ptr(), n_gt, d_off.data_ptr(), g_off.data_ptr(),
                                                     p_off.data_ptr(), G, total, eps_coplanar, eps_nonzero, iou.data_ptr(),
                                                     nbad.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream(dev)), launches=5)
            out = iou[:total].cpu().numpy()
            bad = nbad.tolist()
    if bad[0]:
        print('Warning: skipping {:d} non-coplanar boxes at eval.'.format(int(bad[0])))
    if bad[1]:
        print('Warning: skipping {:d} zero volume boxes at eval.'.format(int(bad[1])))
    res = [out[pair_off[i]:pair_off[i + 1]].reshape(int(nd[i]), int(ng[i])) for i in range(G)]
    return (res, bad) if return_bad_counts else res


def iou2d_xywh(d, g):
    """pycocotools maskUtils.iou(d, g, iscrowd=0) for [x, y, w, h] boxes (omni3d_evaluation.py:1399,1423)."""
    d, g = np.asarray(d, np.float64).reshape(-1, 4), np.asarray(g, np.float64).reshape(-1, 4)
    if len(d) == 0 or len(g) == 0:
        return []
    iw = np.minimum(d[:, None, 0] + d[:, None, 2], g[None, :, 0] + g[None, :, 2]) - np.maximum(d[:, None, 0], g[None, :, 0])
    ih = np.minimum(d[:, None, 1] + d[:, None, 3], g[None, :, 1] + g[None, :, 3]) - np.maximum(d[:, None, 1], g[None, :, 1])
    inter = np.clip(iw, 0, None) * np.clip(ih, 0, None)
    union = (d[:, 2] * d[:, 3])[:, None] + (g[:, 2] * g[:, 3])[None, :] - inter
    return inter / union


def compute_ious_3d(dts, gts, img_ids, cat_ids, max_dets, use_cats=True, eval_prox=False, proximity_thresh=0.3):
    """The reference's `self.ious = {(imgId, catId): self.computeIoU(imgId, catId) ...}` (omni3d_evaluation.py:1339-1343) in
    3D mode.  dts / gts: {(imgId, catId): [ {"score", "bbox3D" (8x3), "bbox" [x,y,w,h], ...}, ... ]} like self._dts / self._gts.
    -> {(imgId, catId): [] | (ious (n,m) ndarray | [], in_prox)}, every 3D IoU coming from ONE segmented launch."""
    cats = list(cat_ids) if use_cats else [-1]
    keys, D, Gs = [], [], []
    for img in img_ids:
        for cat in cats:
            if use_cats:
                gt, dt = gts.get((img, cat), []), dts.get((img, cat), [])
            else:
                gt = [x for c in cat_ids for x in gts.get((img, c), [])]
                dt = [x for c in cat_ids for x in dts.get((img, c), [])]
            inds = np.argsort([-d["score"] for d in dt], kind="mergesort")
            dt = [dt[i] for i in inds][: max_dets]
            keys.append((img, cat)); D.append(dt); Gs.append(gt)
    run = [i for i in range(len(keys)) if len(D[i]) > 0 and len(Gs[i]) > 0]
    mats = box3d_overlap_segmented([[d["bbox3D"] for d in D[i]] for i in run], [[g["bbox3D"] for g in Gs[i]] for i in run]) \
        if run else []
    by = dict(zip(run, mats))
    out = {}
    for i, k in enumerate(keys):
        if len(D[i]) == 0 and len(Gs[i]) == 0:
            out[k] = []
            continue
        ious = by.get(i, [])
        in_prox = None
        if eval_prox:
            i2 = iou2d_xywh([d["bbox"] for d in D[i]], [g["bbox"] for g in Gs[i]])
            in_prox = [] if isinstance(i2, list) else i2 > proximity_thresh
        out[k] = (ious, in_prox)
    return out
