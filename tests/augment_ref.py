"""numpy restatement of the training augmentations before the resize (parse_data(mode='train'),
utils/data_utils.py:140-165 of the reference) and of the flip after it: OpenCV's two 8-bit HSV conversions, every
random draw in the reference's order, and the pixel chain mix-up -> brightness -> BGR2HSV -> hue / saturation / value
-> clip -> HSV2BGR -> expand -> crop.  What csrc/augment.cu (yb_augment_batch, yb_flip_batch) is checked against, next
to the reference-generated goldens of tests/golden/make_golden_augment.py.

BGR2HSV is OpenCV's integer path (modules/imgproc/src/color_hsv.simd.hpp, OpenCV 4.13): 12-bit reciprocal tables
sdiv[v] = round(255 * 4096 / v) and hdiv[d] = round(180 * 4096 / (6 d)), rounded half to even, H in [0, 180).
HSV2BGR is its float path: h * (6 / 180), s / 255, v / 255, the six-sector table with 1 - s f and 1 - s (1 - f) as
fused multiply-adds, then channel * 255 to uint8: truncated in the vector code (each row's first floor(W / 32) * 32
pixels in the AVX2 build), rounded half to even in the scalar tail.  Every other float32 operation rounds on its own.
The box-only crop code (random_crop_with_constraints) is the package's, checked directly on the goldens."""
from __future__ import annotations

import random

import numpy as np

from yolov3_tensorflow_b200.utils.data_aug import random_crop_with_constraints  # host-only box code, checked on goldens

F32 = np.float32
HSV_SHIFT = 12


def _tables():
    i = np.arange(1, 256, dtype=np.float64)
    sdiv = np.zeros(256, np.int64)
    hdiv = np.zeros(256, np.int64)
    sdiv[1:] = np.rint((255 << HSV_SHIFT) / i)
    hdiv[1:] = np.rint((180 << HSV_SHIFT) / (6.0 * i))
    return sdiv, hdiv


SDIV, HDIV = _tables()


def bgr2hsv(img):
    """cv2.cvtColor(img, cv2.COLOR_BGR2HSV) for uint8 [..., 3]."""
    p = np.asarray(img, np.uint8).astype(np.int64)
    b, g, r = p[..., 0], p[..., 1], p[..., 2]
    v = np.maximum(np.maximum(b, g), r)
    diff = v - np.minimum(np.minimum(b, g), r)
    half = 1 << (HSV_SHIFT - 1)
    s = (diff * SDIV[v] + half) >> HSV_SHIFT
    h = np.where(v == r, g - b, np.where(v == g, b - r + 2 * diff, r - g + 4 * diff))
    h = (h * HDIV[diff] + half) >> HSV_SHIFT
    h = np.where(h < 0, h + 180, h)
    return np.stack([h, s, v], -1).astype(np.uint8)


# sector -> (b, g, r) indices into (v, v (1 - s), v (1 - s f), v (1 - s (1 - f)))
_SECTORS = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])


SIMD_PIXELS = 32      # HSV2BGR's vector block in OpenCV's x86-64 build (AVX2: 32 uint8 lanes)


def _one_minus_product(a, b):
    """float32 fma(-a, b, 1): the product is exact in float64, and over the uint8 HSV domain the sum rounds once
    (checked against cv2 on every value by tests/test_augment_host.py)."""
    return (1.0 - a.astype(np.float64) * b.astype(np.float64)).astype(F32)


def hsv2bgr(img):
    """cv2.cvtColor(img, cv2.COLOR_HSV2BGR) for uint8 [H, W, 3] (H in OpenCV's [0, 180) range).  Each row's first
    floor(W / 32) * 32 pixels go through OpenCV's vector code, which truncates channel * 255; the rest through its
    scalar code, which rounds half to even."""
    p = np.asarray(img, np.uint8)
    h = p[..., 0].astype(F32) * F32(6.0 / 180.0)
    s = p[..., 1].astype(F32) * F32(1.0 / 255.0)
    v = p[..., 2].astype(F32) * F32(1.0 / 255.0)
    sector = np.floor(h)
    f = (h - sector).astype(F32)
    sector = sector.astype(np.int64) % 6
    one = F32(1.0)
    tab = np.stack([v, v * (one - s), v * _one_minus_product(s, f), v * _one_minus_product(s, one - f)], -1)
    out = np.take_along_axis(tab.astype(F32), _SECTORS[sector], -1) * F32(255.0)
    w = p.shape[-2]
    simd = (np.arange(w) < w - w % SIMD_PIXELS)[:, None]
    return np.clip(np.where(simd, np.trunc(out), np.rint(out)), 0, 255).astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------------------
# Draws.  One dict per image; `None` means the branch was not taken.
# ---------------------------------------------------------------------------------------------------------------------

def draw_color(brightness_delta=32, hue_vari=18, sat_vari=0.5, val_vari=0.5):
    """random_color_distort's draws (utils/data_aug.py:220-271): brightness, the order coin, then value / saturation /
    hue (or saturation / hue / value), each a p = 0.5 coin and, when it lands above 0.5, its amount."""
    d = {"bright": None, "hue": None, "sat": None, "val": None}
    if np.random.uniform(0, 1) > 0.5:
        d["bright"] = int(np.random.uniform(-brightness_delta, brightness_delta))

    def hue():
        if np.random.uniform(0, 1) > 0.5:
            d["hue"] = int(np.random.randint(-hue_vari, hue_vari))

    def sat():
        if np.random.uniform(0, 1) > 0.5:
            d["sat"] = 1 + np.random.uniform(-sat_vari, sat_vari)

    def val():
        if np.random.uniform(0, 1) > 0.5:
            d["val"] = 1 + np.random.uniform(-val_vari, val_vari)

    for op in ((val, sat, hue) if np.random.randint(0, 2) else (sat, hue, val)):
        op()
    return d


def draw_expand(h, w, max_ratio=4, keep_ratio=True):
    """random_expand's draws -> (canvas h, canvas w, off_y, off_x)."""
    rx = random.uniform(1, max_ratio)
    ry = rx if keep_ratio else random.uniform(1, max_ratio)
    oh, ow = int(h * ry), int(w * rx)
    off_y = random.randint(0, oh - h)
    off_x = random.randint(0, ow - w)
    return oh, ow, off_y, off_x


def draw_flip(px=0.5, py=0):
    """random_flip's two coins -> (horizontal, vertical)."""
    return bool(np.random.uniform(0, 1) < px), bool(np.random.uniform(0, 1) < py)


# ---------------------------------------------------------------------------------------------------------------------
# Pixels
# ---------------------------------------------------------------------------------------------------------------------

def mix_pixels(img1, img2, r):
    """mix_up's image: float32 img1 * r stored, img2 * (1 - r) added where it lies, truncated to uint8."""
    h, w = max(img1.shape[0], img2.shape[0]), max(img1.shape[1], img2.shape[1])
    acc = np.zeros((h, w, 3), F32)
    acc[:img1.shape[0], :img1.shape[1]] = img1.astype(F32) * F32(r)
    acc[:img2.shape[0], :img2.shape[1]] += img2.astype(F32) * F32(1.0 - r)
    return acc.astype(np.uint8)


def color_pixels(img, d):
    """random_color_distort's pixels for the draws d of draw_color."""
    x = np.asarray(img, np.uint8)
    if d["bright"] is not None:
        x = np.clip(x.astype(F32) + F32(d["bright"]), 0, 255).astype(np.uint8)
    hsv = bgr2hsv(x).astype(F32)
    if d["hue"] is not None:
        hsv[..., 0] = np.remainder(hsv[..., 0] + F32(d["hue"]), F32(180))
    if d["sat"] is not None:
        hsv[..., 1] *= F32(d["sat"])
    if d["val"] is not None:
        hsv[..., 2] *= F32(d["val"])
    return hsv2bgr(np.clip(hsv, 0, 255).astype(np.uint8))


def expand_pixels(img, oh, ow, off_y, off_x, fill=0):
    out = np.full((oh, ow, 3), fill, np.uint8)
    out[off_y: off_y + img.shape[0], off_x: off_x + img.shape[1]] = img
    return out


def flip_pixels(img, horizontal, vertical=False):
    if horizontal:
        img = img[:, ::-1]
    if vertical:
        img = img[::-1]
    return np.ascontiguousarray(img)


def flip_boxes(bbox, width, height, horizontal, vertical=False):
    """random_flip's box lines: x' = W - x (y' = H - y) with min and max swapped, in the boxes' dtype."""
    b = bbox.copy()
    if horizontal:
        b[:, 0], b[:, 2] = width - bbox[:, 2], width - bbox[:, 0]
    if vertical:
        b2 = b.copy()
        b[:, 1], b[:, 3] = height - b2[:, 3], height - b2[:, 1]
    return b


def train_image(img1, boxes1, labels1, img2=None, boxes2=None, labels2=None):
    """parse_data(mode='train') for one image up to the resize, drawing from np.random / random in its order ->
    dict(img uint8 crop, boxes, labels (the reference's, not cut to the kept boxes), crop, expand, color, mix, interp,
    flip).  boxes are float32 [N, 5] with a weight column of 1, or float64 after a mix-up, as the reference has them."""
    rec = {"mix": None, "expand": None}
    if img2 is None:
        img = np.asarray(img1, np.uint8)
        boxes = np.concatenate([np.asarray(boxes1, F32).reshape(-1, 4), np.ones((len(boxes1), 1), F32)], 1)
        labels = np.asarray(labels1, np.int64)
    else:
        r = np.random.beta(1.5, 1.5)
        r = max(0, min(1, r))
        rec["mix"] = r
        img = mix_pixels(np.asarray(img1, np.uint8), np.asarray(img2, np.uint8), r)
        b1 = np.asarray(boxes1, F32).reshape(-1, 4)
        b2 = np.asarray(boxes2, F32).reshape(-1, 4)
        boxes = np.concatenate([np.concatenate([b1, np.full((len(b1), 1), r)], 1),
                                np.concatenate([b2, np.full((len(b2), 1), 1.0 - r)], 1)], 0)
        labels = np.concatenate([np.asarray(labels1, np.int64), np.asarray(labels2, np.int64)])
    rec["color"] = draw_color()
    img = color_pixels(img, rec["color"])
    if np.random.uniform(0, 1) > 0.5:
        oh, ow, oy, ox = draw_expand(*img.shape[:2])
        rec["expand"] = (oh, ow, oy, ox)
        img = expand_pixels(img, oh, ow, oy, ox)
        boxes[:, :2] += (ox, oy)
        boxes[:, 2:4] += (ox, oy)
    h, w = img.shape[:2]
    boxes, crop = random_crop_with_constraints(boxes, (w, h))
    x0, y0, cw, ch = crop
    rec["crop"] = crop
    rec["img"] = np.ascontiguousarray(img[y0: y0 + ch, x0: x0 + cw])
    rec["boxes"], rec["labels"] = boxes, labels
    rec["interp"] = int(np.random.randint(0, 5))
    rec["flip"] = draw_flip(0.5)[0]
    return rec
