"""Golden vectors for k-means anchors, produced by the REFERENCE's own get_kmeans.py (iou, avg_iou, translate_boxes,
kmeans, parse_anno, get_kmeans), unmodified.  np.random.seed is replaced by a call with a fixed seed, so the initial
draw is np.random.RandomState(seed).choice(rows, k, replace=False); np.argmin is wrapped to record every iteration's
assignment.  Inputs are regenerated in the tests from the stored seeds (tests/kmeans_ref.py).
Run in the build container only:  python tests/golden/make_golden_kmeans.py"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from tests import kmeans_ref as K  # noqa: E402
# a checkout of wizyoung/YOLOv3_TensorFlow, named by $YOLOV3_TF_REFERENCE
REF = os.environ["YOLOV3_TF_REFERENCE"]
sys.path.insert(0, REF)
import get_kmeans as ref  # noqa: E402

MAX_ITERS = 1000          # the reference never returns once a cluster is empty; the cases are chosen so none is

# tag: (generator, box seed, rows, k, init seed)
CASES = {
    "a": ("float", 1, 2000, 9, 11),
    "b1": ("int", 2, 5000, 1, 21),
    "b2": ("int", 2, 5000, 2, 22),
    "b6": ("int", 2, 5000, 6, 26),
    "b9": ("int", 2, 5000, 9, 29),
    "b12": ("int", 2, 5000, 12, 32),
    "c": ("same", 0, 50, 3, 7),
}


def boxes_of(gen, seed, rows):
    if gen == "float":
        return K.gen_float_boxes(seed, rows)
    if gen == "int":
        return K.gen_int_boxes(seed, rows)
    return np.tile(np.array([[20.0, 30.0]]), (rows, 1))


class Recorder:
    def __init__(self, seed):
        self.seed, self.assigns = seed, []
        self._seed, self._argmin = np.random.seed, np.argmin

    def __enter__(self):
        seed_fn, argmin = self._seed, self._argmin

        def fixed_seed(*args, **kwargs):
            seed_fn(self.seed)

        def recording_argmin(*args, **kwargs):
            r = argmin(*args, **kwargs)
            if kwargs.get("axis") == 1:
                self.assigns.append(np.array(r))
                if len(self.assigns) > MAX_ITERS:
                    raise RuntimeError("reference kmeans does not converge (empty cluster?)")
            return r
        np.random.seed, np.argmin = fixed_seed, recording_argmin
        return self

    def __exit__(self, *exc):
        np.random.seed, np.argmin = self._seed, self._argmin


def main():
    out = {}
    for tag, (gen, bseed, rows, k, iseed) in CASES.items():
        boxes = boxes_of(gen, bseed, rows)
        # the restatement must not meet an empty cluster (the reference would never return)
        K.kmeans(boxes, k, iseed)
        with Recorder(iseed) as rec:
            clusters = ref.kmeans(boxes.copy(), k)                                       # REFERENCE
        with Recorder(iseed):
            anchors, ave = ref.get_kmeans(boxes.copy(), k)                               # REFERENCE
        out[f"{tag}_cfg"] = np.asarray([{"float": 0, "int": 1, "same": 2}[gen], bseed, rows, k, iseed], np.int64)
        out[f"{tag}_assign"] = np.stack(rec.assigns).astype(np.int8)
        out[f"{tag}_clusters"] = clusters
        out[f"{tag}_avg_iou"] = np.float64(ref.avg_iou(boxes, clusters))                 # REFERENCE
        out[f"{tag}_anchors"] = np.asarray(anchors, np.int64)
        out[f"{tag}_ave_iou"] = np.float64(ave)
        print(tag, "iterations", len(rec.assigns), "avg_iou", ave, "anchors", anchors)
    # single-box iou, including the error for a zero-area box
    out["iou_box"] = np.asarray([13.5, 40.25])
    out["iou"] = ref.iou(out["iou_box"], K.gen_float_boxes(3, 9))                          # REFERENCE
    # parse_anno on a generated train.txt
    out["anno_seed"] = np.int64(5)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "train.txt")
        with open(path, "w") as f:
            f.write(K.gen_train_txt(5))
        out["anno_416"] = ref.parse_anno(path, target_size=[416, 416])                   # REFERENCE
        out["anno_none"] = ref.parse_anno(path, target_size=None)                         # REFERENCE
    # translate_boxes
    out["xyxy_seed"] = np.int64(6)
    out["translated"] = ref.translate_boxes(K.gen_xyxy(6, 40))                            # REFERENCE
    np.savez_compressed(os.path.join(HERE, "kmeans.npz"), **out)
    print("wrote", os.path.join(HERE, "kmeans.npz"))


if __name__ == "__main__":
    main()
