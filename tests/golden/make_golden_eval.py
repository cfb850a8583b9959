"""Golden vectors for the evaluation callers of gpu_nms (SURVEY.md 8f N4), produced by the REFERENCE's own
utils/eval_utils.py: evaluate_on_gpu (driven through a stand-in session whose run() is the oracle's gpu_nms — the same
TF-NMS restatement make_golden.py injects), get_preds_gpu, voc_eval / voc_ap.  Inputs are regenerated in the tests from
the stored seeds.  Run in the build container only:  python tests/golden/make_golden_eval.py"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.modules.setdefault("tensorflow", types.ModuleType("tensorflow"))
if "Inf" not in np.__dict__:
    np.Inf = np.inf                      # the reference predates NumPy 2 (utils/eval_utils.py:376 uses np.Inf)
from oracle import yolov3_oracle as O  # noqa: E402
from tests.synth import gen_eval_case  # noqa: E402
# a checkout of wizyoung/YOLOv3_TensorFlow, named by $YOLOV3_TF_REFERENCE
REF = os.environ["YOLOV3_TF_REFERENCE"]
sys.path.insert(0, REF)
from utils import eval_utils as ref  # noqa: E402

NMS = dict(max_boxes=20, score_thresh=0.3, nms_thresh=0.45)


class Sess:                                   # sess.run(gpu_nms_op, feed_dict={boxes_flag: ..., scores_flag: ...})
    def __init__(self, cn):
        self.cn = cn

    def run(self, op, feed_dict):
        b, s = feed_dict["boxes"], feed_dict["scores"]
        r = O.gpu_nms(np.asarray(b, np.float32), np.asarray(s, np.float32), self.cn, NMS["max_boxes"], NMS["score_thresh"], NMS["nms_thresh"])
        return r[0], r[1], r[2]


def main():
    out = {}
    for tag, (seed, n, w, h, cn) in {"a": (5, 4, 160, 128, 20), "b": (9, 3, 96, 96, 80)}.items():
        y_pred, y_true, _ = gen_eval_case(seed, n, w, h, cn)
        tp, tr, pr = ref.evaluate_on_gpu(Sess(cn), None, "boxes", "scores", y_pred, y_true, cn, 0.5, calc_now=False)   # REFERENCE
        rec, prec = ref.evaluate_on_gpu(Sess(cn), None, "boxes", "scores", y_pred, y_true, cn, 0.5, calc_now=True)
        out[f"ev_{tag}_cfg"] = np.asarray([seed, n, w, h, cn], np.int64)
        out[f"ev_{tag}_tp"] = np.asarray([tp[i] for i in range(cn)], np.int64)
        out[f"ev_{tag}_true"] = np.asarray([tr[i] for i in range(cn)], np.int64)
        out[f"ev_{tag}_pred"] = np.asarray([pr[i] for i in range(cn)], np.int64)
        out[f"ev_{tag}_rp"] = np.asarray([rec, prec], np.float64)
        preds = []
        for i in range(n):
            preds += ref.get_preds_gpu(Sess(cn), None, "boxes", "scores", [100 + i], [p[i:i + 1] for p in y_pred])     # REFERENCE
        out[f"pr_{tag}"] = np.asarray([[float(v) for v in row] for row in preds], np.float64).reshape(-1, 7)
        # voc_eval on these predictions against a gt_dict built from the same ground truth
        _, _, gts = gen_eval_case(seed, n, w, h, cn)
        gt_dict = {100 + i: [[float(v) for v in b[:4]] + [int(l)] for b, l in zip(*gts[i])] for i in range(n)}
        res = []
        for c in range(cn):
            for m07 in (False, True):
                gd = {k: [list(o) for o in v] for k, v in gt_dict.items()}
                r = ref.voc_eval(gd, preds, c, iou_thres=0.5, use_07_metric=m07)                                        # REFERENCE
                res.append([c, int(m07)] + [float(v) for v in r])
        out[f"voc_{tag}"] = np.asarray(res, np.float64)
    np.savez_compressed(os.path.join(HERE, "eval.npz"), **out)
    print("wrote eval.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
