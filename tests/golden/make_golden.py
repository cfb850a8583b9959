"""Generate tests/golden/*.npz by running the REFERENCE'S OWN Python sources
(the reference's model.py, utils/layer_utils.py, utils/nms_utils.py,
utils/data_utils.py, utils/misc_utils.py) over the numpy-backed TensorFlow shim
(tf_shim.py).  Needs a checkout of the reference ($YOLOV3_TF_REFERENCE), not a GPU:

    python tests/golden/make_golden.py

The .npz files are committed; tests/test_oracle_golden.py checks oracle/ against them
and the -m gpu tests check the CUDA path against them.  Inputs are regenerated in the
tests from the seeds stored next to the outputs (numpy default_rng / PCG64 streams are
stable across numpy versions), the big tensors (weights) are never stored.
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import tf_shim  # noqa: E402
from tests.synth import gen_inputs, gen_fms  # noqa: E402
from oracle import yolov3_oracle as O  # noqa: E402  (parameter/input generators + TF-kernel restatement of NMS)

tf, slim = tf_shim.install(nms_fn=O.tf_nms_cpu)
# a checkout of wizyoung/YOLOv3_TensorFlow, named by $YOLOV3_TF_REFERENCE
REF = os.environ["YOLOV3_TF_REFERENCE"]
sys.path.insert(0, REF)
import model as ref_model  # noqa: E402
from utils import nms_utils as ref_nms  # noqa: E402
from utils import data_utils as ref_data  # noqa: E402
from utils import misc_utils as ref_misc  # noqa: E402

ANCHORS = ref_misc.parse_anchors(os.path.join(REF, "data", "yolo_anchors.txt"))
assert np.array_equal(ANCHORS, O.COCO_ANCHORS)


def gen_ytrue(seed, n, h, w, class_num, max_boxes=12, empty_first=False):
    rng = np.random.default_rng(seed)
    ys = [[], [], []]
    gts = []
    for i in range(n):
        boxes, labels = O.synth_gt(rng, w, h, class_num, max_boxes)
        boxes[:, 4] = rng.uniform(0.5, 1.0, boxes.shape[0]).astype(np.float32)  # mix-up weights
        if empty_first and i == 0:
            boxes, labels = boxes[:0], labels[:0]
        y = ref_data.process_box(boxes, labels, [w, h], class_num, ANCHORS)      # REFERENCE code
        for j in range(3):
            ys[j].append(y[j])
        gts.append((boxes, labels))
    return [np.stack(y, 0) for y in ys], gts


def main():
    out = {}
    # ---------------- 1. forward wiring (model.py:30-80 + utils/layer_utils.py) ----------------
    C = 80
    n, h, w = 2, 64, 96   # non-square on purpose: catches h/w swaps
    params = O.make_params(C, seed=11, random_bn=True)
    x = gen_inputs(12, n, h, w)
    m = ref_model.yolov3(C, ANCHORS, use_static_shape=False)
    slim.weights = iter(params)
    fms = m.forward(x, is_training=False)
    boxes, confs, probs = m.predict(fms)
    np.savez_compressed(os.path.join(HERE, "forward_infer.npz"), seed_params=11, seed_x=12, shape=[n, h, w],
                        fm1=fms[0], fm2=fms[1], fm3=fms[2], boxes=boxes, confs=confs, probs=probs)
    slim.weights = iter(params); slim.updated_stats = []
    m2 = ref_model.yolov3(C, ANCHORS, batch_norm_decay=0.99, use_static_shape=False)
    fms_t = m2.forward(x, is_training=True)
    st = slim.updated_stats
    np.savez_compressed(os.path.join(HERE, "forward_train.npz"), seed_params=11, seed_x=12, shape=[n, h, w],
                        decay=0.99, fm1=fms_t[0], fm2=fms_t[1], fm3=fms_t[2],
                        mean_first=st[0][0], var_first=st[0][1], mean_last=st[-1][0], var_last=st[-1][1],
                        n_stats=len(st))

    # ---------------- 2. decode (model.py:82-190) on random logits, 2 class counts ----------------
    for tag, cn, (n, h, w) in (("c80", 80, (2, 96, 64)), ("c20", 20, (1, 64, 64))):
        f = gen_fms(21, n, h, w, cn)
        mm = ref_model.yolov3(cn, ANCHORS, use_static_shape=False)
        mm.img_size = tf.shape(np.zeros((n, h, w, 3)))[1:3]
        b, c, p = mm.predict(f)
        xy, bx, cl, pl = mm.reorg_layer(f[0], ANCHORS[6:9])
        np.savez_compressed(os.path.join(HERE, f"decode_{tag}.npz"), seed=21, shape=[n, h, w], class_num=cn,
                            boxes=b, confs=c, probs=p, xy_offset=xy, reorg_boxes=bx)

    # ---------------- 3. loss (model.py:192-365) ----------------
    for tag, cn, (n, h, w), empty in (("a", 80, (3, 96, 64), True), ("b", 20, (2, 64, 64), False)):
        f = gen_fms(31, n, h, w, cn, scale=1.0)
        y_true, gts = gen_ytrue(32, n, h, w, cn, empty_first=empty)
        rec = dict(seed_fm=31, seed_gt=32, shape=[n, h, w], class_num=cn, empty_first=empty,
                   y_true_13=y_true[0], y_true_26=y_true[1], y_true_52=y_true[2])
        for ls in (False, True):
            for fo in (False, True):
                mm = ref_model.yolov3(cn, ANCHORS, use_label_smooth=ls, use_focal_loss=fo, use_static_shape=False)
                mm.img_size = tf.shape(np.zeros((n, h, w, 3)))[1:3]
                losses = mm.compute_loss(f, y_true)
                rec[f"loss_ls{int(ls)}_fo{int(fo)}"] = np.asarray(losses, np.float64)
        # one IoU table straight from box_iou (model.py:307-345)
        mm.img_size = tf.shape(np.zeros((n, h, w, 3)))[1:3]
        _, pb, _, _ = mm.reorg_layer(f[1], ANCHORS[3:6])
        valid = y_true[1][n - 1][..., 0:4][y_true[1][n - 1][..., 4] > 0]
        rec["iou_scale2_lastimg"] = mm.box_iou(pb[n - 1], valid)
        np.savez_compressed(os.path.join(HERE, f"loss_{tag}.npz"), **rec)

    # ---------------- 4. NMS (utils/nms_utils.py) ----------------
    rng = np.random.default_rng(41)
    B, cn = 600, 6
    cx, cy = rng.uniform(0, 128, B), rng.uniform(0, 128, B)
    bw, bh = np.exp(rng.uniform(np.log(4), np.log(64), B)), np.exp(rng.uniform(np.log(4), np.log(64), B))
    bx = np.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1).astype(np.float32)
    sc = (rng.random((B, cn)) * rng.random((B, cn))).astype(np.float32)
    sc[:, 4] = 0.0                                # a class with no candidate
    sc[10:20, 2] = sc[10, 2]                      # exact ties -> lower index first
    gb, gs, gl = ref_nms.gpu_nms(bx[None], sc[None], cn, max_boxes=20, score_thresh=0.3, nms_thresh=0.45)
    cb, cs, cl = ref_nms.cpu_nms(bx[None], sc[None], cn, max_boxes=20, score_thresh=0.3, iou_thresh=0.45)
    keep = ref_nms.py_nms(bx, sc[:, 0], max_boxes=30, iou_thresh=0.5)
    np.savez_compressed(os.path.join(HERE, "nms.npz"), seed=41, boxes_in=bx, scores_in=sc,
                        gpu_boxes=gb, gpu_scores=gs, gpu_labels=gl,
                        cpu_boxes=cb, cpu_scores=cs, cpu_labels=cl, py_keep=np.asarray(keep, np.int64))

    # ---------------- 5. process_box (utils/data_utils.py:51-115) ----------------
    y_true, gts = gen_ytrue(51, 2, 128, 160, 80, max_boxes=30)
    np.savez_compressed(os.path.join(HERE, "process_box.npz"), seed=51, shape=[2, 128, 160],
                        boxes0=gts[0][0], labels0=gts[0][1], boxes1=gts[1][0], labels1=gts[1][1],
                        y13=y_true[0], y26=y_true[1], y52=y_true[2])
    print("golden vectors written to", HERE)
    for fn in sorted(os.listdir(HERE)):
        if fn.endswith(".npz"):
            print(f"  {fn}: {os.path.getsize(os.path.join(HERE, fn)) / 1024:.1f} KiB")


if __name__ == "__main__":
    main()
