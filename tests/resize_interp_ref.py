"""numpy restatement of OpenCV 4.13's uint8 3-channel `cv2.resize` for INTER_CUBIC (2), INTER_AREA (3) and
INTER_LANCZOS4 (4), and of the per-axis tables it builds (modules/imgproc/src/resize.cpp).  What yb_resize_tables and
yb_resize_batch_interp (csrc/preprocess.cu) are checked against, next to the reference-generated goldens of
tests/golden/make_golden_resize_interp.py.

  * INTER_CUBIC / INTER_LANCZOS4: the separable generic path.  Source coordinate f = (float)((d + 0.5) * scale - 0.5),
    s = floor(f), f -= s; 4 (A = -0.75) or 8 float32 coefficients of f rounded to int16 at 11 bits (half to even);
    taps s - k/2 + 1 + j clamped to the image; an int32 horizontal pass.  The vertical pass of Lanczos4 is int32
    (sum + 2^21) >> 22, saturated.  The vertical pass of cubic is OpenCV's SIMD VResizeCubicVec_32s8u on each row's
    first 8 * floor(3 W / 8) values (float32 products with beta * 2^-22, summed S3 + S2, + S1, + S0 outermost last,
    round half to even, saturate) and the scalar int32 (sum + 2^21) >> 22 on the rest.  This is OpenCV's own code:
    the default cv2 build sends uint8 INTER_CUBIC through Intel IPP, which differs by at most 1.
  * INTER_AREA, both axes shrinking by integers: a block mean, (a + b + c + d + 2) >> 2 for 2 x 2 and
    rint(sum * (1.f / area)) otherwise.  Both axes shrinking, not by integers: computeResizeAreaTab's (index, float
    alpha) runs, a float32 horizontal sum per source row and a float32 vertical sum in table order, then rint.
    Otherwise: the bilinear fixed-point path (tests/resize_ref.py) with area-mode coefficients
    s = floor(d * scale), f = (float)((d + 1) - (s + 1) * inv_scale), f = f <= 0 ? 0 : f - floor(f).
  * Same size in and out: a copy, for every interpolation."""
from __future__ import annotations

import math

import numpy as np

from tests import resize_ref as R

F32 = np.float32
CUBIC, AREA, LANCZOS4 = 2, 3, 4


def _scale(dst_size, src_size):
    inv = dst_size / src_size                        # cv::resize: inv_scale = (double)dsize / ssize
    return 1.0 / inv, inv


def cubic_coeffs(x):
    """interpolateCubic(x) in float32, A = -0.75."""
    x = F32(x)
    A = F32(-0.75)
    x1 = F32(x + F32(1))
    c0 = F32(F32(F32(F32(F32(A * x1) - F32(-3.75)) * x1) + F32(-6.0)) * x1) - F32(-3.0)
    c1 = F32(F32(F32(F32(F32(1.25) * x) - F32(2.25)) * x) * x) + F32(1)
    y = F32(F32(1) - x)
    c2 = F32(F32(F32(F32(F32(1.25) * y) - F32(2.25)) * y) * y) + F32(1)
    c3 = F32(F32(F32(F32(1) - c0) - c1) - c2)
    return [c0, c1, c2, c3]


_S45 = 0.70710678118654752440084436210485
_CS = ((1, 0), (-_S45, -_S45), (0, 1), (_S45, -_S45), (-1, 0), (_S45, _S45), (0, -1), (-_S45, _S45))


def lanczos4_coeffs(x):
    """interpolateLanczos4(x): float32 coefficients from double sin / cos (math.sin / math.cos are the C library's),
    normalised by the reciprocal of their float32 sum; a tap at distance < 1e-6 takes 1e30 before normalising."""
    x = F32(x)
    x3 = F32(x + F32(3))
    y0 = float(-x3) * math.pi * 0.25
    s0, c0 = math.sin(y0), math.cos(y0)
    c = []
    total = F32(0)
    for i in range(8):
        yi = F32(x3 - F32(i))
        if abs(yi) >= F32(1e-6):
            y = float(-yi) * math.pi * 0.25
            v = F32((_CS[i][0] * s0 + _CS[i][1] * c0) / (y * y))
        else:
            v = F32(1e30)
        c.append(v)
        total = F32(total + v)
    inv = F32(F32(1) / total)
    return [F32(v * inv) for v in c]


def coef11(c):
    """saturate_cast<short>(c * INTER_RESIZE_COEF_SCALE): round half to even."""
    return int(np.clip(np.rint(F32(F32(c) * F32(2048))), -32768, 32767))


def generic_table(dst_size, src_size, interp):
    """(taps int64 [dst, k] clamped source indices, coefs int32 [dst, k]) of cubic (k = 4) or Lanczos4 (k = 8)."""
    ksize = 4 if interp == CUBIC else 8
    scale, _ = _scale(dst_size, src_size)
    fn = cubic_coeffs if interp == CUBIC else lanczos4_coeffs
    taps = np.zeros((dst_size, ksize), np.int64)
    coefs = np.zeros((dst_size, ksize), np.int32)
    for d in range(dst_size):
        f = F32((d + 0.5) * scale - 0.5)
        s = int(math.floor(f))
        f = F32(f - F32(s))
        coefs[d] = [coef11(c) for c in fn(f)]
        taps[d] = np.clip(np.arange(ksize) + s - ksize // 2 + 1, 0, src_size - 1)
    return taps, coefs


def area_linear_table(dst_size, src_size, clamp_fraction):
    """(s0, s1, c0, c1) of the bilinear path with INTER_AREA's coefficients (any axis grows)."""
    scale, inv = _scale(dst_size, src_size)
    s = np.zeros(dst_size, np.int64)
    f = np.zeros(dst_size, F32)
    for d in range(dst_size):
        sd = int(math.floor(d * scale))
        fd = F32((d + 1) - (sd + 1) * inv)
        fd = F32(0) if fd <= 0 else F32(fd - F32(math.floor(fd)))
        s[d], f[d] = sd, fd
    if clamp_fraction:                               # x: past the last column, one source pixel with weight 1
        hi = s >= src_size - 1
        f[hi] = F32(0)
        s[hi] = src_size - 1
    c0 = np.rint((F32(1.0) - f) * F32(2048.0)).astype(np.int32)
    c1 = np.rint(f * F32(2048.0)).astype(np.int32)
    return np.clip(s, 0, src_size - 1), np.clip(s + 1, 0, src_size - 1), c0, c1


def area_table(dst_size, src_size):
    """computeResizeAreaTab: list of (dst index, src index, float32 alpha) in OpenCV's order."""
    scale, _ = _scale(dst_size, src_size)
    tab = []
    for dx in range(dst_size):
        fsx1 = dx * scale
        fsx2 = fsx1 + scale
        cell = min(scale, src_size - fsx1)
        sx1, sx2 = math.ceil(fsx1), math.floor(fsx2)
        sx2 = min(sx2, src_size - 1)
        sx1 = min(sx1, sx2)
        if sx1 - fsx1 > 1e-3:
            tab.append((dx, sx1 - 1, F32((sx1 - fsx1) / cell)))
        for sx in range(sx1, sx2):
            tab.append((dx, sx, F32(1.0 / cell)))
        if fsx2 - sx2 > 1e-3:
            tab.append((dx, sx2, F32(min(min(fsx2 - sx2, 1.0), cell) / cell)))
    return tab


def area_mode(dst_h, dst_w, src_h, src_w):
    """'fast' (integer shrink on both axes), 'float' (both shrink) or 'linear' (any axis grows)."""
    sx, _ = _scale(dst_w, src_w)
    sy, _ = _scale(dst_h, src_h)
    ix, iy = int(round(sx)), int(round(sy))
    if sx >= 1 and sy >= 1:
        if abs(sx - ix) < np.finfo(np.float64).eps and abs(sy - iy) < np.finfo(np.float64).eps:
            return "fast"
        return "float"
    return "linear"


def _padded(tab, dst_size):
    """Runs of (index, alpha) per destination index, padded with alpha 0 to a rectangle."""
    k = max(sum(1 for t in tab if t[0] == d) for d in range(dst_size))
    idx = np.zeros((dst_size, k), np.int64)
    alpha = np.zeros((dst_size, k), F32)
    fill = np.zeros(dst_size, np.int64)
    for d, s, a in tab:
        idx[d, fill[d]], alpha[d, fill[d]] = s, a
        fill[d] += 1
    return idx, alpha


def _area(img, new_w, new_h):
    sh, sw = img.shape[:2]
    mode = area_mode(new_h, new_w, sh, sw)
    if mode == "linear":
        x0, x1, cx0, cx1 = area_linear_table(new_w, sw, True)
        y0, y1, cy0, cy1 = area_linear_table(new_h, sh, False)
        s = img.astype(np.int32)
        h = s[:, x0] * cx0[None, :, None] + s[:, x1] * cx1[None, :, None]
        v = ((h[y0] >> 4) * cy0[:, None, None] >> 16) + ((h[y1] >> 4) * cy1[:, None, None] >> 16)
        return np.clip((v + 2) >> 2, 0, 255).astype(np.uint8)
    if mode == "fast":
        kx, ky = sw // new_w, sh // new_h
        blocks = img[: new_h * ky, : new_w * kx].astype(np.int64).reshape(new_h, ky, new_w, kx, 3).sum((1, 3))
        if kx == 2 and ky == 2:
            return ((blocks + 2) >> 2).astype(np.uint8)
        return np.clip(np.rint(blocks.astype(F32) * F32(F32(1) / F32(kx * ky))), 0, 255).astype(np.uint8)
    xi, xa = _padded(area_table(new_w, sw), new_w)
    yi, ya = _padded(area_table(new_h, sh), new_h)
    s = img.astype(F32)
    buf = s[:, xi[:, 0]] * xa[None, :, 0, None]
    for k in range(1, xi.shape[1]):                  # buf[dx] + S[sx] * alpha, in table order
        buf = buf + s[:, xi[:, k]] * xa[None, :, k, None]
    acc = ya[:, 0, None, None] * buf[yi[:, 0]]
    for k in range(1, yi.shape[1]):                  # sum += beta * buf, in table order
        acc = acc + ya[:, k, None, None] * buf[yi[:, k]]
    return np.clip(np.rint(acc), 0, 255).astype(np.uint8)


def _hpass(img, taps, coefs):
    s = img.astype(np.int64)
    return sum(s[:, taps[:, k]] * coefs[None, :, k, None] for k in range(taps.shape[1]))      # [sh, new_w, 3]


def cubic_vertical(rows, beta, width):
    """VResizeCubic<uchar> for one output row: rows int [4, width] horizontal sums, beta the 4 int16 coefficients."""
    rows = rows.astype(np.int64)
    out = np.empty(width, np.int64)
    nv = width // 8 * 8                              # VResizeCubicVec_32s8u: 8 values per step (128-bit v_int16)
    if nv:
        b = [F32(F32(bk) * F32(1.0 / (2048 * 2048))) for bk in beta]
        f = rows[:, :nv].astype(F32)
        acc = f[3] * b[3]
        acc = f[2] * b[2] + acc
        acc = f[1] * b[1] + acc
        acc = f[0] * b[0] + acc
        out[:nv] = np.rint(np.clip(acc, -2.0 ** 31, 2.0 ** 31 - 128)).astype(np.int64)
    t = rows[:, nv:]
    out[nv:] = (t[0] * beta[0] + t[1] * beta[1] + t[2] * beta[2] + t[3] * beta[3] + (1 << 21)) >> 22
    return np.clip(out, 0, 255).astype(np.uint8)


def _generic(img, new_w, new_h, interp):
    sh, sw = img.shape[:2]
    xt, xc = generic_table(new_w, sw, interp)
    yt, yc = generic_table(new_h, sh, interp)
    h = _hpass(img, xt, xc)                          # int32 in OpenCV; int64 here (no sum overflows int32)
    if interp == LANCZOS4:
        v = sum(h[yt[:, k]] * yc[:, k, None, None] for k in range(8))
        return np.clip((v + (1 << 21)) >> 22, 0, 255).astype(np.uint8)
    hf = h.reshape(sh, new_w * 3)
    out = np.empty((new_h, new_w * 3), np.uint8)
    for d in range(new_h):
        out[d] = cubic_vertical(hf[yt[d]], yc[d], new_w * 3)
    return out.reshape(new_h, new_w, 3)


def cv2_resize(img, new_w, new_h, interp):
    """cv2.resize(img, (new_w, new_h), interpolation=interp) for uint8 [H, W, 3], interp 0..4 (cubic with IPP off)."""
    img = np.asarray(img, np.uint8)
    if interp in (0, 1):
        return R.cv2_resize(img, new_w, new_h, interp)
    if img.shape[:2] == (new_h, new_w):
        return img.copy()
    if interp == AREA:
        return _area(img, new_w, new_h)
    if interp in (CUBIC, LANCZOS4):
        return _generic(img, new_w, new_h, interp)
    raise ValueError(f"interp {interp}: not an OpenCV interpolation in 0..4")


def letterbox_resize(img, new_w, new_h, interp):
    """utils/data_aug.py:274-293 -> (uint8 padded image, resize_ratio, dw, dh)."""
    ori_h, ori_w = img.shape[:2]
    ratio, rw, rh, dw, dh = R.letterbox_geometry(ori_h, ori_w, new_w, new_h)
    padded = np.full((new_h, new_w, 3), 128, np.uint8)
    padded[dh: rh + dh, dw: rw + dw, :] = cv2_resize(img, rw, rh, interp)
    return padded, ratio, dw, dh


def resize_image(img, new_w, new_h, interp, letterbox):
    """The uint8 image of resize_with_bbox (utils/data_aug.py:296-318)."""
    if letterbox:
        return letterbox_resize(img, new_w, new_h, interp)[0]
    return cv2_resize(img, new_w, new_h, interp)


def preprocess(img, new_w, new_h, letterbox, interp):
    """One image of yb_resize_batch_interp: float32 RGB [new_h, new_w, 3] and its params row."""
    x = R.normalize(resize_image(img, new_w, new_h, interp, letterbox))
    if letterbox:
        ratio, _, _, dw, dh = R.letterbox_geometry(img.shape[0], img.shape[1], new_w, new_h)
        return x, (ratio, float(dw), float(dh))
    return x, (img.shape[1] / float(new_w), img.shape[0] / float(new_h), 0.0)
