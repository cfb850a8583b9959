"""Golden vectors for the device-side pre-processing (SURVEY.md 8f N3), produced by the REFERENCE's own code:
  * utils/data_aug.letterbox_resize (cv2 nearest-neighbour, interp=0) + the BGR->RGB / float32 / 255 lines of
    test_single_image.py:44-46, on small synthetic uint8 images (wide, tall, up- and down-scaling);
  * utils/data_utils.process_box on box lists built to COLLIDE (several boxes in one (scale, cell, anchor) slot, with
    different classes and mix-up weights), where the list order decides what survives.
Run in the build container only:  python tests/golden/make_golden_preprocess.py"""
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
from utils import data_aug, data_utils  # noqa: E402

ANCHORS = np.reshape(np.asarray(open(os.path.join(REF, "data", "yolo_anchors.txt")).read().split(","), np.float32), [-1, 2])


def main():
    out = {}
    rng = np.random.default_rng(41)
    cases = [(75, 100, 128, 96), (60, 33, 64, 64), (33, 60, 96, 64), (200, 310, 96, 96), (17, 23, 160, 128)]   # src h, w -> new w, h
    out["letterbox_cases"] = np.asarray(cases, np.int64)
    for i, (sh, sw, nw, nh) in enumerate(cases):
        img = rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8)
        pad, ratio, dw, dh = data_aug.letterbox_resize(img, nw, nh)                 # REFERENCE code
        x = cv2.cvtColor(pad, cv2.COLOR_BGR2RGB)                                   # test_single_image.py:44
        x = np.asarray(x, np.float32)                                              # :45
        x = x[np.newaxis, :] / 255.                                                # :46
        out[f"lb_src{i}"] = img
        out[f"lb_out{i}"] = x.astype(np.float32)
        out[f"lb_meta{i}"] = np.asarray([ratio, dw, dh], np.float64)
    # process_box with collisions: 3 images, W x H = 160 x 128
    W, H, C = 160, 128, 80
    gts = []
    for i in range(3):
        v = [14, 9, 1][i]
        cx = rng.uniform(8, W - 8, v); cy = rng.uniform(8, H - 8, v)
        bw = np.exp(rng.uniform(np.log(6), np.log(150), v)); bh = np.exp(rng.uniform(np.log(6), np.log(120), v))
        boxes = np.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2, rng.uniform(0.3, 1.0, v)], 1).astype(np.float32)
        labels = rng.integers(0, C, v).astype(np.int64)
        if v >= 9:      # force collisions: copies of earlier boxes (same cell, same best anchor) with other classes / weights
            for dst, src in ((5, 1), (7, 1), (8, 3)):
                boxes[dst, :4] = boxes[src, :4] + np.float32(0.25)
                labels[dst] = (labels[src] + 7 + dst) % C
        gts.append((boxes, labels))
    ys = [[], [], []]
    for boxes, labels in gts:
        y = data_utils.process_box(boxes, labels, [W, H], C, ANCHORS)              # REFERENCE code
        for j in range(3):
            ys[j].append(y[j])
    out["pb_shape"] = np.asarray([W, H, C], np.int64)
    for i, (b, l) in enumerate(gts):
        out[f"pb_boxes{i}"] = b
        out[f"pb_labels{i}"] = l
    # stored sparse: (flat index, value) of the entries that differ from the default fill (0, mix weight 1)
    for j, name in enumerate(("y13", "y26", "y52")):
        y = np.stack(ys[j], 0)
        base = np.zeros_like(y); base[..., -1] = 1.0
        idx = np.flatnonzero(y != base)
        out[f"pb_{name}_shape"] = np.asarray(y.shape, np.int64)
        out[f"pb_{name}_idx"] = idx.astype(np.int64)
        out[f"pb_{name}_val"] = y.reshape(-1)[idx]
    np.savez_compressed(os.path.join(HERE, "preprocess.npz"), **out)
    print("wrote preprocess.npz:", {k: v.shape for k, v in out.items() if k.startswith("pb_y")})


if __name__ == "__main__":
    main()
