"""numpy restatement of the evaluation input path: OpenCV's uint8 3-channel `cv2.resize` (INTER_NEAREST and
INTER_LINEAR), `letterbox_resize` / `resize_with_bbox` (utils/data_aug.py:274-318), the BGR->RGB / float32 / 255 lines
of test_single_image.py:44-46 and its detection back-mapping (:64-70).  What the device kernels of csrc/preprocess.cu
(yb_resize_batch, yb_resize_boxes, yb_restore_boxes) are checked against, next to the reference-generated goldens of
tests/golden/make_golden_resize.py.

INTER_LINEAR is OpenCV's fixed-point path (modules/imgproc/src/resize.cpp, OpenCV 4.13): 11-bit coefficients rounded
half to even, a 32-bit horizontal pass and the SIMD vertical pass
  v = (((h0 >> 4) * c0y >> 16) + ((h1 >> 4) * c1y >> 16) + 2) >> 2.
x sources are clamped with their fraction zeroed; y keeps its fraction and only the row indices are clamped.  OpenCV
does not promise INTER_LINEAR is bit-stable across builds (INTER_LINEAR_EXACT is the stable mode), so this restates the
build the goldens were made with."""
from __future__ import annotations

import numpy as np

F32 = np.float32


def nearest_index(dst_size, src_size):
    """resizeNN: min(floor(d * (1 / (dst / src))), src - 1) in double."""
    ifs = 1.0 / (dst_size / src_size)
    return np.minimum(np.floor(np.arange(dst_size) * ifs).astype(np.int64), src_size - 1)


def linear_coeffs(dst_size, src_size, clamp_fraction):
    """(s0, s1, c0, c1) per destination coordinate: source indices (clamped) and 11-bit coefficients."""
    scale = 1.0 / (dst_size / src_size)
    f = ((np.arange(dst_size, dtype=np.float64) + 0.5) * scale - 0.5).astype(F32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(F32)).astype(F32)
    if clamp_fraction:                       # x: the border columns take one source pixel with weight 1
        lo, hi = s < 0, s >= src_size - 1
        f[lo | hi] = F32(0.0)
        s[lo] = 0
        s[hi] = src_size - 1
    c0 = np.rint((F32(1.0) - f) * F32(2048.0)).astype(np.int32)           # saturate_cast<short>: half to even
    c1 = np.rint(f * F32(2048.0)).astype(np.int32)
    s0 = np.clip(s, 0, src_size - 1)
    s1 = np.clip(s + 1, 0, src_size - 1)
    return s0, s1, c0, c1


def cv2_resize(img, new_w, new_h, interp):
    """cv2.resize(img, (new_w, new_h), interpolation=interp) for uint8 [H, W, 3], interp 0 (nearest) or 1 (linear)."""
    img = np.asarray(img, np.uint8)
    sh, sw = img.shape[:2]
    if interp == 0:
        return img[nearest_index(new_h, sh)][:, nearest_index(new_w, sw)]
    if interp != 1:
        raise ValueError(f"interp {interp}: only 0 (nearest) and 1 (linear) are restated")
    x0, x1, cx0, cx1 = linear_coeffs(new_w, sw, True)
    y0, y1, cy0, cy1 = linear_coeffs(new_h, sh, False)
    s = img.astype(np.int32)
    h = s[:, x0] * cx0[None, :, None] + s[:, x1] * cx1[None, :, None]       # [sh, new_w, 3] int32
    h0, h1 = h[y0] >> 4, h[y1] >> 4
    v = ((h0 * cy0[:, None, None]) >> 16) + ((h1 * cy1[:, None, None]) >> 16)
    return np.clip((v + 2) >> 2, 0, 255).astype(np.uint8)


def letterbox_geometry(ori_h, ori_w, new_w, new_h):
    """(resize_ratio, resize_w, resize_h, dw, dh) of letterbox_resize (utils/data_aug.py:279-289)."""
    ratio = min(new_w / ori_w, new_h / ori_h)
    rw, rh = int(ratio * ori_w), int(ratio * ori_h)
    return ratio, rw, rh, int((new_w - rw) / 2), int((new_h - rh) / 2)


def letterbox_resize(img, new_w, new_h, interp):
    """utils/data_aug.py:274-293 -> (uint8 padded image, resize_ratio, dw, dh)."""
    ori_h, ori_w = img.shape[:2]
    ratio, rw, rh, dw, dh = letterbox_geometry(ori_h, ori_w, new_w, new_h)
    padded = np.full((new_h, new_w, 3), 128, np.uint8)
    padded[dh: rh + dh, dw: rw + dw, :] = cv2_resize(img, rw, rh, interp)
    return padded, ratio, dw, dh


def normalize(img_bgr_u8):
    """cvtColor(BGR2RGB) -> np.float32 -> / 255. (float32 division)."""
    return (np.asarray(img_bgr_u8[..., ::-1], F32) / F32(255.0)).astype(F32)


def preprocess(img, new_w, new_h, letterbox, interp):
    """One image of yb_resize_batch: float32 RGB [new_h, new_w, 3] and its params row
    (resize_ratio, dw, dh) for letterbox, (ori_w / new_w, ori_h / new_h, 0) for stretch."""
    if letterbox:
        padded, ratio, dw, dh = letterbox_resize(img, new_w, new_h, interp)
        return normalize(padded), (ratio, float(dw), float(dh))
    ori_h, ori_w = img.shape[:2]
    return normalize(cv2_resize(img, new_w, new_h, interp)), (ori_w / float(new_w), ori_h / float(new_h), 0.0)


def resize_boxes(boxes, ori_h, ori_w, new_w, new_h, letterbox):
    """resize_with_bbox's box lines (utils/data_aug.py:301-318), float32 boxes [V, >=4] with numpy 2 (NEP 50) scalar
    promotion: the Python-float ratio and the int sizes act as float32."""
    b = np.array(boxes, F32, copy=True)
    if letterbox:
        ratio, _, _, dw, dh = letterbox_geometry(ori_h, ori_w, new_w, new_h)
        b[:, [0, 2]] = b[:, [0, 2]] * F32(ratio) + F32(dw)
        b[:, [1, 3]] = b[:, [1, 3]] * F32(ratio) + F32(dh)
    else:
        b[:, [0, 2]] = b[:, [0, 2]] / F32(ori_w) * F32(new_w)
        b[:, [1, 3]] = b[:, [1, 3]] / F32(ori_h) * F32(new_h)
    return b


def restore_boxes(boxes, params_row, letterbox):
    """test_single_image.py:64-70: network-input boxes [V, 4] float32 -> source-image coordinates."""
    b = np.array(boxes, F32, copy=True)
    a0, a1, a2 = params_row
    if letterbox:
        b[:, [0, 2]] = (b[:, [0, 2]] - F32(a1)) / F32(a0)
        b[:, [1, 3]] = (b[:, [1, 3]] - F32(a2)) / F32(a0)
    else:
        b[:, [0, 2]] *= F32(a0)
        b[:, [1, 3]] *= F32(a1)
    return b
