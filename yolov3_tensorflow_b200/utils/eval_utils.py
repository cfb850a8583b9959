"""utils/eval_utils.py of the reference, the callers of gpu_nms (SURVEY.md 8f N4): per-batch recall / precision
(`evaluate_on_gpu`, :142-234), detection lists for mAP (`get_preds_gpu`, :237-261) and the PASCAL-VOC metric
(`voc_ap`, `voc_eval`, :311-423).  The reference runs one `sess.run(gpu_nms_op)` per image; here the whole batch goes
through ONE batched NMS call on the device (utils.nms_utils.batched_nms_raw) and only the kept detections come back
to the host, where the bookkeeping (a few hundred boxes) stays numpy like the reference's."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .. import _lib
from .._lib import lib, check, ptr, stream_handle
from .nms_utils import batched_nms_raw


def calc_iou(pred_boxes, true_boxes):
    """IoU matrix [N, V] of corner-format boxes [N,4] x [V,4] (utils/eval_utils.py:13-45; +1e-10 in the denominator)."""
    p = np.asarray(pred_boxes)[:, None, :]
    t = np.asarray(true_boxes)[None, :, :]
    wh = np.maximum(np.minimum(p[..., 2:], t[..., 2:]) - np.maximum(p[..., :2], t[..., :2]), 0.)
    inter = wh[..., 0] * wh[..., 1]
    pa = (p[..., 2] - p[..., 0]) * (p[..., 3] - p[..., 1])
    ta = (t[..., 2] - t[..., 0]) * (t[..., 3] - t[..., 1])
    return inter / (pa + ta - inter + 1e-10)


def gt_from_y_true(y_true, i):
    """Ground truth of image i out of the three y_true tensors (utils/eval_utils.py:153-182):
    -> (labels list [V], boxes [V,4] xmin,ymin,xmax,ymax float64).  Objects = cells with a non-zero class vector,
    label = argmax of it, visited scale 13 -> 26 -> 52 in row-major cell order."""
    labels, boxes = [], []
    for y in y_true:
        yi = y[i]
        yi = yi.detach().cpu().numpy() if isinstance(yi, torch.Tensor) else np.asarray(yi)
        probs = yi[..., 5:-1]
        mask = probs.sum(axis=-1) > 0
        labels += np.argmax(probs[mask], axis=-1).tolist()
        boxes += yi[..., 0:4][mask].tolist()
    tb = np.array(boxes, dtype=np.float64).reshape(-1, 4)
    out = np.empty_like(tb)
    out[:, 0:2] = tb[:, 0:2] - tb[:, 2:4] / 2.
    out[:, 2:4] = out[:, 0:2] + tb[:, 2:4]
    return labels, out


def matched_gt(pred_boxes, pred_labels, true_boxes, true_labels, iou_thresh):
    """Indices of the ground-truth boxes counted as true positives (utils/eval_utils.py:200-226): a prediction
    qualifies when its best-overlapping gt box has IoU > iou_thresh and the same label; every gt index is counted
    once however many predictions hit it (the reference's confidence bookkeeping never removes an index)."""
    if len(pred_labels) == 0 or len(true_labels) == 0:
        return np.zeros((0,), np.int64)
    iou = calc_iou(pred_boxes, true_boxes)
    best = np.argmax(iou, axis=-1)
    ok = (iou[np.arange(len(best)), best] > iou_thresh) & (np.asarray(true_labels)[best] == np.asarray(pred_labels))
    return np.unique(best[ok])


def _nms_batch(y_pred, num_classes, max_boxes, score_thresh, nms_thresh):
    boxes, confs, probs = y_pred[0], y_pred[1], y_pred[2]
    dev = boxes.device if isinstance(boxes, torch.Tensor) and boxes.is_cuda else torch.device(f"cuda:{torch.cuda.current_device()}")
    tb = torch.as_tensor(boxes, dtype=torch.float32).to(dev)
    tc = torch.as_tensor(confs, dtype=torch.float32).to(dev)
    tp = torch.as_tensor(probs, dtype=torch.float32).to(dev)
    scores = tc * tp                                   # pred_confs * pred_probs (utils/eval_utils.py:195,252); off the hot path
    ob, os_, ol, oi, cnt = batched_nms_raw(tb, scores, num_classes, max_boxes, score_thresh, nms_thresh)
    ks = cnt.cpu().tolist()                            # one host synchronisation for the whole batch
    ob, os_, ol = ob.cpu().numpy(), os_.cpu().numpy(), ol.cpu().numpy()
    return [(ob[i, :k], os_[i, :k], ol[i, :k]) for i, k in enumerate(ks)]


def evaluate_on_gpu(y_pred, y_true, num_classes, iou_thresh=0.5, calc_now=True, max_boxes=50, score_thresh=0.5,
                    nms_thresh=0.5):
    """utils/eval_utils.py:142-234.  y_pred = [boxes [N,B,4], confs [N,B,1], probs [N,B,C]] (model.predict),
    y_true = [y_true_13, y_true_26, y_true_52].  max_boxes / score_thresh / nms_thresh are the arguments the reference
    bakes into its gpu_nms_op (train.py:76).  -> (recall, precision), or the three per-class dicts if not calc_now."""
    n = int(y_true[0].shape[0])
    true_d = {i: 0 for i in range(num_classes)}
    pred_d = {i: 0 for i in range(num_classes)}
    tp_d = {i: 0 for i in range(num_classes)}
    dets = _nms_batch(y_pred, num_classes, max_boxes, score_thresh, nms_thresh)
    for i in range(n):
        t_labels, t_boxes = gt_from_y_true(y_true, i)
        for c in t_labels:
            true_d[c] += 1
        p_boxes, _, p_labels = dets[i]
        for c in p_labels.tolist():
            pred_d[c] += 1
        for t in matched_gt(p_boxes, p_labels, t_boxes, t_labels, iou_thresh):
            tp_d[t_labels[t]] += 1
    if not calc_now:
        return tp_d, true_d, pred_d
    tp = sum(tp_d.values())
    return tp / (sum(true_d.values()) + 1e-6), tp / (sum(pred_d.values()) + 1e-6)


def get_preds_gpu(image_ids, y_pred, num_classes, max_boxes=50, score_thresh=0.5, nms_thresh=0.5):
    """utils/eval_utils.py:237-261 for a whole batch: -> [[image_id, x_min, y_min, x_max, y_max, score, label], ...]
    (the reference handles image_ids[0] only; with one image the result is identical)."""
    dets = _nms_batch(y_pred, num_classes, max_boxes, score_thresh, nms_thresh)
    out = []
    for img_id, (b, s, l) in zip(image_ids, dets):
        for k in range(len(l)):
            out.append([img_id, b[k, 0], b[k, 1], b[k, 2], b[k, 3], s[k], l[k]])
    return out


def voc_ap(rec, prec, use_07_metric=False):
    """utils/eval_utils.py:311-340: 11-point VOC07 metric or the area under the monotone precision envelope."""
    rec, prec = np.asarray(rec), np.asarray(prec)
    if use_07_metric:
        ap = 0.
        for t in np.arange(0., 1.1, 0.1):
            ap = ap + (np.max(prec[rec >= t]) if np.sum(rec >= t) != 0 else 0) / 11.
        return ap
    mrec = np.concatenate(([0.], rec, [1.]))
    mpre = np.concatenate(([0.], prec, [0.]))
    mpre = np.maximum.accumulate(mpre[::-1])[::-1]
    i = np.where(mrec[1:] != mrec[:-1])[0]
    return np.sum((mrec[i + 1] - mrec[i]) * mpre[i + 1])


def voc_eval(gt_dict, val_preds, classidx, iou_thres=0.5, use_07_metric=False):
    """utils/eval_utils.py:343-423.  gt_dict {img_id: [[x0,y0,x1,y1,label], ...]}, val_preds = get_preds_gpu rows.
    -> (npos, nd, recall, precision, ap) of class `classidx` (VOC '+1 pixel' overlap, a gt box matches once)."""
    recs, npos = {}, 0
    for img_id, objs in gt_dict.items():
        bb = np.array([o[:4] for o in objs if o[-1] == classidx])
        recs[img_id] = (bb, np.zeros(len(bb), bool))
        npos += len(bb)
    pred = [x for x in val_preds if x[-1] == classidx]
    if not pred:
        print('no box, ignore')
        return 1e-6, 1e-6, 0, 0, 0
    order = np.argsort(-np.array([x[-2] for x in pred]))
    nd = len(pred)
    tp, fp = np.zeros(nd), np.zeros(nd)
    for d, j in enumerate(order):
        bb = np.array(pred[j][1:5])
        gt, used = recs[pred[j][0]]
        ovmax, jmax = -np.inf, -1
        if gt.size > 0:
            iw = np.maximum(np.minimum(gt[:, 2], bb[2]) - np.maximum(gt[:, 0], bb[0]) + 1., 0.)
            ih = np.maximum(np.minimum(gt[:, 3], bb[3]) - np.maximum(gt[:, 1], bb[1]) + 1., 0.)
            inter = iw * ih
            uni = (bb[2] - bb[0] + 1.) * (bb[3] - bb[1] + 1.) + (gt[:, 2] - gt[:, 0] + 1.) * (gt[:, 3] - gt[:, 1] + 1.) - inter
            ov = inter / uni
            jmax = int(np.argmax(ov))
            ovmax = ov[jmax]
        if ovmax > iou_thres and not used[jmax]:
            tp[d] = 1.
            used[jmax] = True
        else:
            fp[d] = 1.
    fp, tp = np.cumsum(fp), np.cumsum(tp)
    rec = tp / float(npos)
    prec = tp / np.maximum(tp + fp, np.finfo(np.float64).eps)
    return npos, nd, tp[-1] / float(npos), tp[-1] / float(nd), voc_ap(rec, prec, use_07_metric)


def parse_gt_rec_lines(lines, target_img_size, letterbox_resize=True):
    """utils/eval_utils.py:265-305 on already-parsed annotation rows (img_id, boxes [V,4], labels [V], ori_width,
    ori_height): ground truth mapped into the network's input frame -> gt_dict for voc_eval."""
    new_w, new_h = target_img_size
    gt = {}
    for img_id, boxes, labels, ow, oh in lines:
        objs = []
        for (x0, y0, x1, y1), lab in zip(boxes, labels):
            if letterbox_resize:
                r = min(new_w / ow, new_h / oh)
                dw, dh = int((new_w - int(r * ow)) / 2), int((new_h - int(r * oh)) / 2)
                objs.append([x0 * r + dw, y0 * r + dh, x1 * r + dw, y1 * r + dh, lab])
            else:
                objs.append([x0 * new_w / ow, y0 * new_h / oh, x1 * new_w / ow, y1 * new_h / oh, lab])
        gt[img_id] = objs
    return gt


def pack_gt_rec(gt_dict, image_ids, vmax=None):
    """Ground truth of a batch in parse_gt_rec_lines' format ({img_id: [[x0, y0, x1, y1, label], ...]}) -> padded host
    arrays for VOCEvaluator.add_batch, pinned when CUDA is available: boxes [n, vmax, 4] float64 (the coordinates voc_eval compares
    with), labels [n, vmax] int32, counts [n] int32.  Padding is zero boxes with label -1."""
    objs = [gt_dict.get(i, []) for i in image_ids]
    n = len(objs)
    if n == 0:
        raise ValueError("pack_gt_rec: no images")
    counts = np.asarray([len(o) for o in objs], np.int32)
    vmax = int(vmax or max(1, int(counts.max())))
    if int(counts.max()) > vmax:
        raise ValueError(f"pack_gt_rec: {int(counts.max())} boxes > vmax {vmax}")
    hb = torch.zeros((n, vmax, 4), dtype=torch.float64)
    hl = torch.full((n, vmax), -1, dtype=torch.int32)
    for i, o in enumerate(objs):
        if o:
            hb[i, :len(o)] = torch.from_numpy(np.asarray([r[:4] for r in o], np.float64))
            hl[i, :len(o)] = torch.from_numpy(np.asarray([int(r[-1]) for r in o], np.int32))
    out = (hb, hl, torch.from_numpy(counts))
    return tuple(t.pin_memory() for t in out) if torch.cuda.is_available() else out


class VOCEvaluator:
    """voc_eval for every class of a validation set on the device (libyolob200.so: yb_voc_match, yb_voc_ap).

    add_batch() takes one batch's NMS output as detect_raw / batched_nms_raw return it ([n, C*max_boxes] layout) and
    its ground truth (pack_gt_rec), matches detections to ground truth on the device and appends one 8-byte record
    per detection to a device pool; no detection is copied to the host.  result() sorts the pool and returns, per
    class, what voc_eval(gt_dict, rows, c, iou_thresh, use_07_metric) returns for the get_preds_gpu rows of the same
    batches in the same order, with ties in score ranked in that order (a stable sort; numpy's default sort may order
    ties either way).  Both metrics can be read from one pool."""

    def __init__(self, num_classes, iou_thresh=0.5, device=None):
        self.num_classes = int(num_classes)
        if not 1 <= self.num_classes <= 65535:
            raise ValueError(f"VOCEvaluator: num_classes {num_classes} outside [1, 65535]")
        self.iou_thresh = float(iou_thresh)
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self._pool = torch.empty((1 << 16,), dtype=torch.int64, device=self.device)
        self._class_counts = torch.zeros((self.num_classes, 2), dtype=torch.int64, device=self.device)
        self._size = 0
        self._ws = None

    def reset(self):
        self._size = 0
        self._class_counts.zero_()

    def __len__(self):
        """Detections added so far."""
        return self._size

    def add_batch(self, out_boxes, out_scores, out_labels, counts, gt_boxes, gt_labels, gt_counts):
        """out_boxes [n, cap, 4] float32, out_scores [n, cap] float32, out_labels [n, cap] int32, counts [n] int32 on
        the device (detect_raw / batched_nms_raw output); gt_boxes [n, vmax, 4] float64, gt_labels [n, vmax] int32,
        gt_counts [n] int32, host (copied asynchronously) or device.  One host synchronisation: the batch's detection
        count, read to grow the pool."""
        dev = self.device
        for t in (out_boxes, out_scores, out_labels, counts):
            if not (isinstance(t, torch.Tensor) and t.is_cuda and t.device == dev):
                raise TypeError(f"VOCEvaluator.add_batch: detections must be CUDA tensors on {dev}")
        if (out_boxes.dtype, out_scores.dtype, out_labels.dtype, counts.dtype) != (torch.float32, torch.float32,
                                                                                    torch.int32, torch.int32):
            raise TypeError("VOCEvaluator.add_batch: expects float32 boxes / scores and int32 labels / counts")
        n, cap = int(out_scores.shape[0]), int(out_scores.shape[1])
        if tuple(out_boxes.shape) != (n, cap, 4) or tuple(out_labels.shape) != (n, cap) or tuple(counts.shape) != (n,):
            raise ValueError(f"VOCEvaluator.add_batch: detection shapes {tuple(out_boxes.shape)} / {tuple(out_scores.shape)}"
                             f" / {tuple(out_labels.shape)} / {tuple(counts.shape)}")
        gb = gt_boxes.to(dev, non_blocking=True).contiguous()
        gl = gt_labels.to(dev, non_blocking=True).contiguous()
        gc = gt_counts.to(dev, non_blocking=True).contiguous()
        if gb.dtype != torch.float64 or gl.dtype != torch.int32 or gc.dtype != torch.int32:
            raise TypeError("VOCEvaluator.add_batch: expects float64 gt boxes and int32 gt labels / counts")
        vmax = int(gb.shape[1]) if gb.dim() == 3 else -1
        if tuple(gb.shape) != (n, vmax, 4) or tuple(gl.shape) != (n, vmax) or tuple(gc.shape) != (n,):
            raise ValueError(f"VOCEvaluator.add_batch: gt shapes {tuple(gb.shape)} / {tuple(gl.shape)} / {tuple(gc.shape)}"
                             f" do not match {n} images")
        if vmax > _lib.YB_VOC_MAX_GT:
            raise ValueError(f"VOCEvaluator.add_batch: {vmax} gt boxes per image > {_lib.YB_VOC_MAX_GT}")
        if n == 0:
            return
        ob, os_, ol, oc = out_boxes.contiguous(), out_scores.contiguous(), out_labels.contiguous(), counts.contiguous()
        with torch.cuda.device(dev):
            total = int(oc.clamp(0, cap).sum())               # the one host synchronisation
            need = self._size + total
            if need > self._pool.numel():
                pool = torch.empty((max(need, 2 * self._pool.numel()),), dtype=torch.int64, device=dev)
                pool[:self._size].copy_(self._pool[:self._size])
                self._pool = pool
            check(lib.yb_voc_match(ptr(ob), ptr(os_), ptr(ol), ptr(oc), n, cap, ptr(gb), ptr(gl), ptr(gc), vmax,
                                   self.num_classes, self.iou_thresh, ptr(self._pool), self._size, self._pool.numel(),
                                   ptr(self._class_counts), stream_handle()), "yb_voc_match")
        self._size = need

    def result(self, use_07_metric=False):
        """[(npos, nd, rec, prec, ap)] for classes 0..C-1, as voc_eval returns them ((1e-6, 1e-6, 0, 0, 0) for a class
        without detections)."""
        dev = self.device
        need = C.c_size_t()
        check(lib.yb_voc_ap_workspace_bytes(self._size, self.num_classes, C.byref(need)), "yb_voc_ap_workspace_bytes")
        if self._ws is None or self._ws.numel() < need.value:
            self._ws = torch.empty((max(need.value, 256),), dtype=torch.uint8, device=dev)
        out = torch.empty((self.num_classes, 5), dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            check(lib.yb_voc_ap(ptr(self._pool), self._size, ptr(self._class_counts), self.num_classes,
                                int(bool(use_07_metric)), ptr(self._ws), self._ws.numel(), ptr(out), stream_handle()),
                  "yb_voc_ap")
            res = out.cpu().numpy()
        rows = []
        for npos, nd, rec, prec, ap in res.tolist():
            if nd == 1e-6:
                rows.append((1e-6, 1e-6, 0, 0, 0))
            else:
                rows.append((int(npos), int(nd), np.float64(rec), np.float64(prec), np.float64(ap)))
        return rows

    def summary(self, use_07_metric=False):
        """(mAP, recall, precision) as eval.py:125-137 reports them: AP averaged over the classes, recall weighted by
        npos, precision weighted by nd (AverageMeter.update(val, n) in class order)."""
        sums, cnts = [0., 0., 0.], [0., 0., 0.]
        for npos, nd, rec, prec, ap in self.result(use_07_metric):
            for k, (v, w) in enumerate(((ap, 1), (rec, npos), (prec, nd))):
                sums[k] += v * w
                cnts[k] += w
        return tuple(s / float(c) for s, c in zip(sums, cnts))
