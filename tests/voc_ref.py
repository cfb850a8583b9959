"""Test oracles for the device VOC evaluator (utils.eval_utils.VOCEvaluator).

voc_eval_stable is utils.eval_utils.voc_eval with one change: detections are ranked by a STABLE argsort of -score, so
equal scores keep row order.  That is the order the device evaluator defines; numpy's default sort may put ties
either way.  voc_from_flags is the same computation vectorised, for sets whose TP flags are known by construction."""
import numpy as np

from yolov3_tensorflow_b200.utils.eval_utils import voc_ap


def _stable_counts(gt_dict, val_preds, classidx, iou_thres):
    recs, npos = {}, 0
    for img_id, objs in gt_dict.items():
        bb = np.array([o[:4] for o in objs if o[-1] == classidx])
        recs[img_id] = (bb, np.zeros(len(bb), bool))
        npos += len(bb)
    pred = [x for x in val_preds if x[-1] == classidx]
    if not pred:
        return npos, None, None
    order = np.argsort(-np.array([x[-2] for x in pred]), kind="stable")
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
    return npos, tp, fp


def _finish(npos, tp, fp, use_07_metric):
    if tp is None:
        return 1e-6, 1e-6, 0, 0, 0
    nd = len(tp)
    fp, tp = np.cumsum(fp), np.cumsum(tp)
    rec = tp / float(npos)
    prec = tp / np.maximum(tp + fp, np.finfo(np.float64).eps)
    return npos, nd, tp[-1] / float(npos), tp[-1] / float(nd), voc_ap(rec, prec, use_07_metric)


def voc_eval_stable(gt_dict, val_preds, classidx, iou_thres=0.5, use_07_metric=False):
    return _finish(*_stable_counts(gt_dict, val_preds, classidx, iou_thres), use_07_metric)


def voc_eval_stable_all(gt_dict, val_preds, num_classes, iou_thres=0.5):
    """voc_eval_stable of every class under both metrics, matching each class once -> (area results, 11-point results)."""
    by_class = {c: [] for c in range(num_classes)}
    for r in val_preds:
        by_class[int(r[-1])].append(r)
    area, p11 = [], []
    with np.errstate(divide="ignore", invalid="ignore"):
        for c in range(num_classes):
            counts = _stable_counts(gt_dict, by_class[c], c, iou_thres)
            area.append(_finish(*counts, False))
            p11.append(_finish(*counts, True))
    return area, p11


def voc_from_flags(labels, scores, tp_flags, npos, num_classes, use_07_metric=False):
    """Per-class voc_eval result from detections in insertion order whose TP flags are already known."""
    labels, scores, tp_flags = np.asarray(labels), np.asarray(scores, np.float32), np.asarray(tp_flags)
    out = []
    for c in range(num_classes):
        sel = labels == c
        if not sel.any():
            out.append((1e-6, 1e-6, 0, 0, 0))
            continue
        t = tp_flags[sel][np.argsort(-scores[sel], kind="stable")].astype(np.float64)
        tp, fp = np.cumsum(t), np.cumsum(1. - t)
        with np.errstate(divide="ignore", invalid="ignore"):
            rec = tp / float(npos[c])
            prec = tp / np.maximum(tp + fp, np.finfo(np.float64).eps)
            out.append((int(npos[c]), int(sel.sum()), tp[-1] / float(npos[c]), tp[-1] / float(sel.sum()),
                        voc_ap(rec, prec, use_07_metric)))
    return out


def rows_from_nms(image_ids, out_boxes, out_scores, out_labels, counts):
    """get_preds_gpu's rows from NMS output held on the host (float32 numpy arrays, like _nms_batch returns)."""
    rows = []
    for img_id, b, s, l, k in zip(image_ids, out_boxes, out_scores, out_labels, counts):
        for j in range(int(k)):
            rows.append([img_id, b[j, 0], b[j, 1], b[j, 2], b[j, 3], s[j], l[j]])
    return rows


def assert_voc_equal(got, want, area_tol=1e-12, use_07_metric=False):
    """npos, nd, rec, prec bit-exact (nan-aware); ap bit-exact for the 11-point metric, within area_tol for the area."""
    assert len(got) == len(want)
    for c, (g, w) in enumerate(zip(got, want)):
        g64, w64 = np.asarray([float(v) for v in g]), np.asarray([float(v) for v in w])
        assert np.array_equal(g64[:4], w64[:4], equal_nan=True), (c, g, w)
        if use_07_metric:
            assert np.array_equal(g64[4:], w64[4:], equal_nan=True), (c, g, w)
        else:
            assert (np.isnan(g64[4]) and np.isnan(w64[4])) or abs(g64[4] - w64[4]) <= area_tol, (c, g, w)
