"""Host-side mirror of the reference's 3D-IoU interface, running on libc3d.so (sm_90a).

    box3d_overlap(boxes_dt, boxes_gt, eps_coplanar=1e-4, eps_nonzero=1e-8) -> iou (N, M)
        == cubercnn/evaluation/omni3d_evaluation.py:106-166 (same name, argument meaning and
        error behaviour: offending dt rows are zeroed and a warning is printed, never raised).
    iou_box3d(boxes1, boxes2) -> (vol, iou)
        == pytorch3d._C.iou_box3d as called at omni3d_evaluation.py:155.

Inputs may be CUDA tensors (used in place) or CPU tensors / arrays (copied to the device, result
returned on the CPU like the reference, which runs this op on the CPU at
omni3d_evaluation.py:1404-1412).
"""
import torch

from . import _lib
from ._lib import ptr, stream

_ws_cache = {}


def _workspace(nbytes, device):
    key = device.index if device.index is not None else torch.cuda.current_device()
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return buf


def _prep(boxes, device):
    if not isinstance(boxes, torch.Tensor):
        boxes = torch.as_tensor(boxes)
    if boxes.dim() != 3 or tuple(boxes.shape[1:]) != (8, 3):
        raise ValueError(f"boxes must be (n, 8, 3), got {tuple(boxes.shape)}")
    return boxes.to(device=device, dtype=torch.float32, non_blocking=True).contiguous()


def _device_of(*ts):
    for t in ts:
        if isinstance(t, torch.Tensor) and t.is_cuda:
            return t.device
    if not torch.cuda.is_available():
        raise _lib.C3DError("omni3d_b200.box3d needs a CUDA device (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def _is_cuda(x):
    return isinstance(x, torch.Tensor) and x.is_cuda


def iou_box3d(boxes1, boxes2, with_counts=False):
    """(N,8,3), (M,8,3) -> vol (N,M), iou (N,M) [, nfaces (N,M) int32] on the input's device."""
    L = _lib.lib()
    dev = _device_of(boxes1, boxes2)
    ret_cpu = not _is_cuda(boxes1)
    with torch.cuda.device(dev):
        b1, b2 = _prep(boxes1, dev), _prep(boxes2, dev)
        N, M = b1.shape[0], b2.shape[0]
        vol = torch.empty((N, M), dtype=torch.float32, device=dev)
        iou = torch.empty((N, M), dtype=torch.float32, device=dev)
        nf = torch.empty((N, M), dtype=torch.int32, device=dev) if with_counts else None
        if N * M > 0:
            ws = _workspace(L.c3d_iou_box3d_workspace_bytes(N, M), dev)
            _lib.check(L.c3d_iou_box3d(ptr(b1), N, ptr(b2), M, ptr(vol), ptr(iou), ptr(nf), ptr(ws),
                                       ws.numel(), stream(dev)), launches=4)
    out = (vol, iou, nf) if with_counts else (vol, iou)
    return tuple(o.cpu() for o in out) if ret_cpu else out


def iou_box3d_paired(boxes1, boxes2, with_counts=False):
    """pair k = (boxes1[k], boxes2[k]) -> vol (n,), iou (n,) [, nfaces (n,)]."""
    L = _lib.lib()
    dev = _device_of(boxes1, boxes2)
    ret_cpu = not _is_cuda(boxes1)
    with torch.cuda.device(dev):
        b1, b2 = _prep(boxes1, dev), _prep(boxes2, dev)
        n = b1.shape[0]
        if b2.shape[0] != n:
            raise ValueError("paired mode needs equally many boxes")
        vol = torch.empty(n, dtype=torch.float32, device=dev)
        iou = torch.empty(n, dtype=torch.float32, device=dev)
        nf = torch.empty(n, dtype=torch.int32, device=dev) if with_counts else None
        if n > 0:
            ws = _workspace(L.c3d_iou_box3d_workspace_bytes(n, 0), dev)
            _lib.check(L.c3d_iou_box3d_paired(ptr(b1), ptr(b2), n, ptr(vol), ptr(iou), ptr(nf), ptr(ws),
                                              ws.numel(), stream(dev)), launches=3)
    out = (vol, iou, nf) if with_counts else (vol, iou)
    return tuple(o.cpu() for o in out) if ret_cpu else out


def box3d_overlap(boxes_dt, boxes_gt, eps_coplanar: float = 1e-4, eps_nonzero: float = 1e-8,
                  return_bad_counts: bool = False):
    """Drop-in for cubercnn.evaluation.omni3d_evaluation.box3d_overlap (:106-166)."""
    L = _lib.lib()
    dev = _device_of(boxes_dt, boxes_gt)
    ret_cpu = not _is_cuda(boxes_dt)
    with torch.cuda.device(dev):
        b1, b2 = _prep(boxes_dt, dev), _prep(boxes_gt, dev)
        N, M = b1.shape[0], b2.shape[0]
        iou = torch.empty((N, M), dtype=torch.float32, device=dev)
        nbad = torch.zeros(2, dtype=torch.int32, device=dev)
        if N > 0:
            ws = _workspace(L.c3d_iou_box3d_workspace_bytes(N, max(M, 1)), dev)
            _lib.check(L.c3d_box3d_overlap(ptr(b1), N, ptr(b2), M, eps_coplanar, eps_nonzero, ptr(iou),
                                           ptr(nbad), ptr(ws), ws.numel(), stream(dev)), launches=5)
        bad = nbad.tolist()   # the reference's .any() checks (:158,162) are host syncs too
    if bad[0]:
        print('Warning: skipping {:d} non-coplanar boxes at eval.'.format(int(bad[0])))
    if bad[1]:
        print('Warning: skipping {:d} zero volume boxes at eval.'.format(int(bad[1])))
    out = iou.cpu() if ret_cpu else iou
    return (out, bad) if return_bad_counts else out
