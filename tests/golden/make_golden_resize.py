"""Golden vectors for the batched evaluation input path (yb_resize_batch, yb_resize_boxes, yb_restore_boxes), produced
by the REFERENCE's own code under OpenCV 4.13:
  * utils/data_aug.letterbox_resize with interp=0 and interp=1;
  * utils/data_aug.resize_with_bbox(interp=1) for letterbox=True and False (parse_data(mode='val'),
    utils/data_utils.py:172), images and boxes, and with interp=0 for the nearest stretch;
  * test_single_image.py's stretch (cv2.resize at its default interpolation) + BGR->RGB / float32 / 255 (:39-46) and
    its two back-mapping branches (:64-70) on detection-like boxes.
Small synthetic images: up- and down-scaling, a 1 x 1 source, an exact 2x downscale, odd sizes, extreme aspect ratios
and non-square targets.  Images are stored as the reference's uint8 results (the float input is that / 255).
Run in the build container only:  YOLOV3_TF_REFERENCE=<checkout> python tests/golden/make_golden_resize.py"""
import os
import sys
import types

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.modules.setdefault("tensorflow", types.ModuleType("tensorflow"))       # utils/*.py import it at module level
# a checkout of wizyoung/YOLOv3_TensorFlow, named by $YOLOV3_TF_REFERENCE
REF = os.environ["YOLOV3_TF_REFERENCE"]
sys.path.insert(0, REF)
from utils import data_aug  # noqa: E402

# src h, src w -> new w, new h
CASES = [(30, 40, 64, 48), (75, 100, 40, 32), (1, 1, 32, 24), (64, 96, 48, 32), (33, 61, 48, 40), (5, 120, 64, 32),
         (110, 4, 32, 64), (50, 50, 64, 32), (41, 23, 37, 53), (2, 3, 64, 64), (96, 64, 32, 32), (1, 7, 24, 40)]


def main():
    out = {"cv2_version": np.asarray(cv2.__version__)}
    rng = np.random.default_rng(2024)
    out["cases"] = np.asarray(CASES, np.int64)
    for i, (sh, sw, nw, nh) in enumerate(CASES):
        img = rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8)
        out[f"src{i}"] = img
        lb0, r0, dw0, dh0 = data_aug.letterbox_resize(img, nw, nh, interp=0)           # REFERENCE code
        lb1, r1, dw1, dh1 = data_aug.letterbox_resize(img, nw, nh, interp=1)
        assert (r0, dw0, dh0) == (r1, dw1, dh1)
        out[f"lb0_{i}"], out[f"lb1_{i}"] = lb0, lb1
        out[f"lb_meta{i}"] = np.asarray([r1, dw1, dh1], np.float64)
        # ground truth as parse_data holds it: float32 [V, 5] with the mix-up weight column
        v = 4
        x0 = rng.uniform(0, sw, v); x1 = rng.uniform(0, sw, v)
        y0 = rng.uniform(0, sh, v); y1 = rng.uniform(0, sh, v)
        gt = np.stack([np.minimum(x0, x1), np.minimum(y0, y1), np.maximum(x0, x1), np.maximum(y0, y1),
                       np.ones(v)], 1).astype(np.float32)
        out[f"gt{i}"] = gt
        im_l, b_l = data_aug.resize_with_bbox(img, gt.copy(), nw, nh, interp=1, letterbox=True)     # REFERENCE code
        im_s, b_s = data_aug.resize_with_bbox(img, gt.copy(), nw, nh, interp=1, letterbox=False)
        im_s0, _ = data_aug.resize_with_bbox(img, gt.copy(), nw, nh, interp=0, letterbox=False)
        assert np.array_equal(im_l, lb1)
        out[f"gt_lb{i}"], out[f"gt_st{i}"] = b_l, b_s
        out[f"st1_{i}"], out[f"st0_{i}"] = im_s, im_s0
        # test_single_image.py:43 (cv2.resize's default interpolation is INTER_LINEAR)
        height_ori, width_ori = img.shape[:2]
        st = cv2.resize(img, (nw, nh))
        assert np.array_equal(st, im_s)
        # detections in the network-input frame, float32 as sess.run returns them; test_single_image.py:64-70
        det = np.sort(rng.uniform(-4, max(nw, nh) + 4, (6, 4)).astype(np.float32).reshape(6, 2, 2), 1).reshape(6, 4)
        det = det[:, [0, 2, 1, 3]].copy()
        out[f"det{i}"] = det
        boxes_ = det.copy()
        boxes_[:, [0, 2]] = (boxes_[:, [0, 2]] - dw1) / r1
        boxes_[:, [1, 3]] = (boxes_[:, [1, 3]] - dh1) / r1
        out[f"det_lb{i}"] = boxes_
        boxes_ = det.copy()
        boxes_[:, [0, 2]] *= (width_ori / float(nw))
        boxes_[:, [1, 3]] *= (height_ori / float(nh))
        out[f"det_st{i}"] = boxes_
    # one float network input exactly as test_single_image.py:43-46 builds it (stretch)
    sh, sw, nw, nh = CASES[4]
    x = cv2.cvtColor(cv2.resize(out["src4"], (nw, nh)), cv2.COLOR_BGR2RGB)
    x = np.asarray(x, np.float32)
    out["x_st4"] = (x[np.newaxis, :] / 255.).astype(np.float32)
    path = os.path.join(HERE, "resize.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path)} bytes, {len(CASES)} cases, OpenCV {cv2.__version__}")


if __name__ == "__main__":
    main()
