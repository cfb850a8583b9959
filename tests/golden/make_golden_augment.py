"""Golden vectors for the training augmentation (yb_augment_batch, yb_flip_batch, utils.data_aug's draws), produced by
the REFERENCE's own utils/data_aug.py under OpenCV 4.13: parse_data(mode='train')'s steps (utils/data_utils.py:
140-165) called in its order from fixed np.random / random seeds — mix_up for paired images, random_color_distort,
the expand coin and random_expand, random_crop_with_constraints and the crop, the interp draw, then
resize_with_bbox(letterbox=True) and random_flip at 64 x 64.  Recorded per image: the crop's pixels, boxes, labels and
window, the drawn interp and flip, the resized and flipped image and boxes, and both RNG states after the image.
Synthetic images of odd sizes, a 1 x 1 and box-less images among them.
Run in the build container only:  YOLOV3_TF_REFERENCE=<checkout> python tests/golden/make_golden_augment.py"""
import os
import random
import sys
import types

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.modules.setdefault("tensorflow", types.ModuleType("tensorflow"))       # utils/*.py import it at module level
REF = os.environ["YOLOV3_TF_REFERENCE"]
sys.path.insert(0, REF)
from utils import data_aug  # noqa: E402

# (h, w, boxes)
SIZES = [(75, 100, 3), (37, 53, 2), (1, 1, 0), (64, 33, 4), (120, 90, 1), (17, 129, 2), (48, 48, 0), (200, 150, 5),
         (33, 65, 3), (90, 41, 2), (5, 300, 1), (160, 96, 2)]
MIX = [None, 3, None, 0, 7, None, None, 1, None, 10, None, 2]        # image i mixed with image MIX[i]
SIZE = 64


def _images_and_boxes():
    rng = np.random.default_rng(77)
    imgs, boxes, labels = [], [], []
    for h, w, v in SIZES:
        imgs.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        x0, x1 = rng.uniform(0, w, v), rng.uniform(0, w, v)
        y0, y1 = rng.uniform(0, h, v), rng.uniform(0, h, v)
        b = np.stack([np.minimum(x0, x1), np.minimum(y0, y1), np.maximum(x0, x1) + 1, np.maximum(y0, y1) + 1], 1)
        boxes.append(b.astype(np.float32).reshape(-1, 4))
        labels.append(rng.integers(0, 20, v).astype(np.int64))
    return imgs, boxes, labels


def main():
    imgs, boxes, labels = _images_and_boxes()
    out = {"cv2_version": np.asarray(cv2.__version__), "numpy_version": np.asarray(np.__version__),
           "sizes": np.asarray(SIZES, np.int64), "mix": np.asarray([-1 if m is None else m for m in MIX], np.int64)}
    for i in range(len(SIZES)):
        out[f"src{i}"], out[f"gt{i}"], out[f"lab{i}"] = imgs[i], boxes[i], labels[i]
    np.random.seed(2026)
    random.seed(1234)
    # NumPy 2 scalars: Python floats, so float32 arrays times them stay float32 (NEP 50)
    assert type(np.random.beta(1.5, 1.5)) is float and type(np.random.uniform(0, 1)) is float
    np.random.seed(2026)
    for i in range(len(SIZES)):
        if MIX[i] is None:                                              # parse_data, utils/data_utils.py:128-132
            img = imgs[i]
            bx = np.concatenate((boxes[i], np.full((len(boxes[i]), 1), 1., np.float32)), axis=-1)
            lab = labels[i]
        else:
            j = MIX[i]
            img, bx = data_aug.mix_up(imgs[i], imgs[j], boxes[i], boxes[j])   # REFERENCE code from here on
            lab = np.concatenate((labels[i], labels[j]))
        img = data_aug.random_color_distort(img)
        if np.random.uniform(0, 1) > 0.5:
            img, bx = data_aug.random_expand(img, bx, 4)
        h, w, _ = img.shape
        bx, crop = data_aug.random_crop_with_constraints(bx, (w, h))
        x0, y0, w, h = crop
        img = img[y0: y0 + h, x0: x0 + w]
        out[f"crop_img{i}"], out[f"boxes{i}"], out[f"labels{i}"] = img, bx, lab
        out[f"crop{i}"] = np.asarray(crop, np.int64)
        interp = np.random.randint(0, 5)
        out[f"interp{i}"] = np.asarray(interp)
        state = np.random.get_state()
        out[f"flip{i}"] = np.asarray(np.random.uniform(0, 1) < 0.5)
        np.random.set_state(state)
        if img.size:
            rimg, rbx = data_aug.resize_with_bbox(img, bx.copy(), SIZE, SIZE, interp=interp, letterbox=True)
            rimg, rbx = data_aug.random_flip(rimg, rbx, px=0.5)
            out[f"final_img{i}"], out[f"final_boxes{i}"] = rimg, rbx
        else:                                                           # cv2.resize rejects an empty crop
            np.random.uniform(0, 1), np.random.uniform(0, 1)
        st = np.random.get_state()
        out[f"np_keys{i}"], out[f"np_pos{i}"] = st[1], np.asarray(st[2])
        out[f"py_state{i}"] = np.asarray(random.getstate()[1], np.int64)
    path = os.path.join(HERE, "augment.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path)} bytes, {len(SIZES)} images, OpenCV {cv2.__version__}, "
          f"NumPy {np.__version__}")


if __name__ == "__main__":
    main()
