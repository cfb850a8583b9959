"""utils/nms_utils.py of the reference, re-hosted: `gpu_nms` runs the sm_90a NMS kernels
(libyolob200.so: yb_nms); `py_nms` / `cpu_nms` keep the reference's numpy semantics
(a *different* algorithm: +1 pixel areas, `<=` keep rule — utils/nms_utils.py:51-123)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .. import _lib
from .._lib import lib, check, ptr, stream_handle

_WS_CACHE = {}


def _workspace(n, B, Cn, mb, device):
    """Scratch for one yb_nms call.  Cached per (device, stream): calls on one stream are ordered, so they may share
    it; calls on different streams get different buffers.  A buffer that has to grow is replaced — the old tensor goes
    back to torch's caching allocator, which keeps it alive until the stream's queued work has used it."""
    need = C.c_size_t()
    check(lib.yb_nms_workspace_bytes(n, B, Cn, mb, C.byref(need)), "yb_nms_workspace_bytes")
    with torch.cuda.device(device):
        key = (str(device), torch.cuda.current_stream().cuda_stream)
    ws = _WS_CACHE.get(key)
    if ws is None or ws.numel() < need.value:
        ws = torch.empty(max(need.value, 256), dtype=torch.uint8, device=device)
        _WS_CACHE[key] = ws
    return ws


def batched_nms_raw(boxes, scores, num_classes, max_boxes, score_thresh, nms_thresh):
    """Device-side result for a batch: boxes [n,B,4], scores [n,B,C] ->
    (out_boxes [n,C*mb,4], out_scores, out_labels, out_indices [n,C*mb], counts [n]) — no host sync."""
    if not (isinstance(boxes, torch.Tensor) and boxes.is_cuda and isinstance(scores, torch.Tensor) and scores.is_cuda):
        raise TypeError("gpu_nms expects CUDA tensors")
    if boxes.dtype != torch.float32 or scores.dtype != torch.float32:
        raise TypeError("gpu_nms expects float32 tensors")
    n = boxes.shape[0]
    boxes = boxes.contiguous()
    scores = scores.contiguous()
    B = boxes.shape[1]
    if boxes.shape != (n, B, 4) or scores.shape != (n, B, num_classes):
        raise ValueError(f"gpu_nms: shapes {tuple(boxes.shape)} / {tuple(scores.shape)} do not match num_classes={num_classes}")
    dev = boxes.device
    cap = num_classes * max(int(max_boxes), 0)
    ob = torch.empty((n, max(cap, 1), 4), dtype=torch.float32, device=dev)
    os_ = torch.empty((n, max(cap, 1)), dtype=torch.float32, device=dev)
    ol = torch.empty((n, max(cap, 1)), dtype=torch.int32, device=dev)
    oi = torch.empty((n, max(cap, 1)), dtype=torch.int32, device=dev)
    cnt = torch.empty((n,), dtype=torch.int32, device=dev)
    ws = _workspace(n, B, num_classes, int(max_boxes), dev)
    with torch.cuda.device(dev):                       # the tensors' device, not whatever device happens to be current
        check(lib.yb_nms(ptr(boxes), ptr(scores), n, B, num_classes, int(max_boxes), float(score_thresh), float(nms_thresh),
                         ptr(ws), ws.numel(), ptr(ob), ptr(os_), ptr(ol), ptr(oi), ptr(cnt), stream_handle()), "yb_nms")
    return ob, os_, ol, oi, cnt


def gpu_nms(boxes, scores, num_classes, max_boxes=50, score_thresh=0.5, nms_thresh=0.5, return_indices=False):
    """utils/nms_utils.py:8-48.  Single image, like the reference (it reshapes to [-1,4]):
    boxes [1,B,4] (or [B,4]) xyxy, scores [1,B,C].  Returns (boxes [K,4], score [K], label [K] int32)
    on the device, classes ascending, descending score inside a class, at most max_boxes PER CLASS.
    return_indices=True appends the original box index of every kept box (not available in the reference).
    Reading K back is the one host synchronisation of this call."""
    if not (isinstance(boxes, torch.Tensor) and isinstance(scores, torch.Tensor)):
        raise TypeError("gpu_nms expects torch CUDA tensors")
    if boxes.numel() % 4 or scores.numel() % num_classes or boxes.numel() // 4 != scores.numel() // num_classes:
        raise ValueError(f"gpu_nms: shapes {tuple(boxes.shape)} / {tuple(scores.shape)} do not match num_classes={num_classes}")
    b = boxes.reshape(1, -1, 4)                    # utils/nms_utils.py:26-27
    s = scores.reshape(1, -1, num_classes)
    ob, os_, ol, oi, cnt = batched_nms_raw(b, s, num_classes, max_boxes, score_thresh, nms_thresh)
    k = int(cnt.item())
    out = (ob[0, :k], os_[0, :k], ol[0, :k])
    if return_indices:
        out = out + (oi[0, :k],)
    return out


def batched_gpu_nms(boxes, scores, num_classes, max_boxes=50, score_thresh=0.5, nms_thresh=0.5):
    """gpu_nms applied independently to every image of a batch (the reference can only do one
    image per call, SURVEY.md F3).  Returns a list of (boxes, score, label, index) per image."""
    ob, os_, ol, oi, cnt = batched_nms_raw(boxes, scores, num_classes, max_boxes, score_thresh, nms_thresh)
    ks = cnt.tolist()
    return [(ob[i, :k], os_[i, :k], ol[i, :k], oi[i, :k]) for i, k in enumerate(ks)]


def py_nms(boxes, scores, max_boxes=50, iou_thresh=0.5):
    """Pure numpy NMS baseline with the reference's semantics (utils/nms_utils.py:51-88)."""
    assert boxes.shape[1] == 4 and len(scores.shape) == 1
    x1, y1, x2, y2 = boxes[:, 0], boxes[:, 1], boxes[:, 2], boxes[:, 3]
    areas = (x2 - x1) * (y2 - y1)
    order = scores.argsort()[::-1]
    keep = []
    while order.size > 0:
        i = order[0]
        keep.append(i)
        rest = order[1:]
        w = np.maximum(0.0, np.minimum(x2[i], x2[rest]) - np.maximum(x1[i], x1[rest]) + 1)
        h = np.maximum(0.0, np.minimum(y2[i], y2[rest]) - np.maximum(y1[i], y1[rest]) + 1)
        inter = w * h
        ovr = inter / (areas[i] + areas[rest] - inter)
        order = rest[np.where(ovr <= iou_thresh)[0]]
    return keep[:max_boxes]


def cpu_nms(boxes, scores, num_classes, max_boxes=50, score_thresh=0.5, iou_thresh=0.5):
    """numpy per-class NMS with the reference's semantics (utils/nms_utils.py:91-123)."""
    boxes = boxes.reshape(-1, 4)
    scores = scores.reshape(-1, num_classes)
    pb, ps, pl = [], [], []
    for i in range(num_classes):
        idx = np.where(scores[:, i] >= score_thresh)
        fb, fs = boxes[idx], scores[:, i][idx]
        if len(fb) == 0:
            continue
        keep = py_nms(fb, fs, max_boxes=max_boxes, iou_thresh=iou_thresh)
        pb.append(fb[keep]); ps.append(fs[keep]); pl.append(np.ones(len(keep), dtype="int32") * i)
    if len(pb) == 0:
        return None, None, None
    return np.concatenate(pb, axis=0), np.concatenate(ps, axis=0), np.concatenate(pl, axis=0)
