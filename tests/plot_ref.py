"""numpy / Python restatement of the OpenCV 4.13 drawing that the reference's plot_one_box does:
cv2.rectangle (LINE_8, any thickness, and filled), cv2.getTextSize and cv2.putText (FONT_HERSHEY_SIMPLEX, LINE_AA,
thickness 1).  Written from OpenCV's documented algorithms, step by step as OpenCV runs them: integer 16.16 fixed
point, Cohen-Sutherland clipping in doubles, the midpoint circle and LineAA's filter and end-point tables.  The font
and the tables come from csrc/hershey_simplex.inc, which is generated from the OpenCV library itself.

It is the reference the device drawing is compared against; line_aa, rectangle and text_segments can be run one
primitive at a time to find where two images part."""
import math
import os
import re

import numpy as np

XY_SHIFT = 16
XY_ONE = 1 << XY_SHIFT
INC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolov3_tensorflow_b200", "csrc",
                   "hershey_simplex.inc")


def _load():
    src = open(INC).read()
    glyphs = [g.replace('\\"', '"').replace("\\\\", "\\")
              for g in re.findall(r'^    "((?:[^"\\]|\\.)*?)\\0" /\*', src, re.M)]
    assert len(glyphs) == 95
    filt = [int(v) for v in re.search(r"YB_AA_FILTER \{(.*)\}", src).group(1).split(",")]
    slope = [int(v) for v in re.search(r"YB_AA_SLOPE_CORR \{(.*)\}", src).group(1).split(",")]
    base = int(re.search(r"YB_HS_BASE_LINE (\d+)", src).group(1))
    cap = int(re.search(r"YB_HS_CAP_LINE (\d+)", src).group(1))
    sin = [float(np.float32(float.fromhex(v.strip().rstrip("f"))))
           for v in re.search(r"YB_SIN_TABLE \{(.*)\}", src).group(1).split(",")]
    assert len(sin) == 451
    return glyphs, filt, slope, base, cap, sin


GLYPHS, FILTER, SLOPE_CORR, BASE_LINE, CAP_LINE, SIN_TABLE = _load()


def tdiv(a, b):
    """C integer division (truncates toward zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def cv_round(v):
    return int(round(v))                       # cvRound: nearest, ties to even (lrint)


def text_codes(label):
    """Characters as putText reads them for FONT_HERSHEY_SIMPLEX: byte by byte of the UTF-8 string; a byte outside
    ' ' .. '~' (every byte of a non-ASCII character, and control characters) draws '?'."""
    return [b if 32 <= b < 127 else ord("?") for b in label.encode("utf-8")]


def text_size(codes, scale, thickness):
    """cv2.getTextSize(text, FONT_HERSHEY_SIMPLEX, scale, thickness)[0] -> (width, height)."""
    view_x = 0.0
    for c in codes:
        g = GLYPHS[c - 32]
        view_x += (ord(g[1]) - ord(g[0])) * scale
    return cv_round(view_x + thickness), cv_round((CAP_LINE + BASE_LINE) * scale + (thickness + 1) // 2)


def line_thickness(h, w, line_thickness=None):
    return line_thickness or int(round(0.002 * max(h, w)))


def label_layout(codes, tl, c1):
    """The reference's label geometry: (t_size, label rectangle corner c2, putText origin, font thickness)."""
    tf = max(tl - 1, 1)
    tw, th = text_size(codes, float(tl) / 3, tf)
    return (tw, th), (c1[0] + tw, c1[1] - th - 3), (c1[0], c1[1] - 2), tf


def fill_rect(img, x0, y0, x1, y1, color):
    """Every pixel of [x0, x1] x [y0, y1] (inclusive, either order) inside the image."""
    h, w = img.shape[:2]
    xa, xb = max(min(x0, x1), 0), min(max(x0, x1), w - 1)
    ya, yb = max(min(y0, y1), 0), min(max(y0, y1), h - 1)
    if xa <= xb and ya <= yb:
        img[ya:yb + 1, xa:xb + 1] = color


def circle_spans(radius):
    """The midpoint circle's filled rows: {dy: half width} (Circle(..., fill=1))."""
    spans = {}
    err, dx, dy, plus, minus = 0, radius, 0, 1, (radius << 1) - 1
    while dx >= dy:
        for r, half in ((dy, dx), (dx, dy)):
            spans[r] = max(spans.get(r, -1), half)
        dy += 1
        err += plus
        plus += 2
        mask = -1 if err > 0 else 0
        err -= minus & mask
        dx += mask
        minus -= mask & 2
    return spans


def fill_circle(img, cx, cy, radius, color):
    for dy, half in circle_spans(radius).items():
        for y in {cy - dy, cy + dy}:
            if 0 <= y < img.shape[0]:
                fill_rect(img, cx - half, y, cx + half, y, color)


def rectangle(img, c1, c2, color, thickness):
    """cv2.rectangle(img, c1, c2, color, thickness) with LINE_8 and shift 0.  The outline is one colour, so its
    pixels are the union of its pieces: per side ThickLine's quad (or the 1-pixel Line), and a filled circle at the
    end of each side (the polyline is closed, so every corner gets one)."""
    if thickness < 0:
        fill_rect(img, c1[0], c1[1], c2[0], c2[1], color)
        return
    pts = [c1, (c2[0], c1[1]), c2, (c1[0], c2[1])]
    p0 = pts[3]
    for p in pts:
        if thickness <= 1:
            fill_rect(img, p0[0], p0[1], p[0], p[1], color)      # an axis-parallel LINE_8 line
        else:
            half = (thickness + 1) // 2        # cvRound(dy * (thickness + odd) * XY_ONE / 2 / |d|), exact here
            if p0[0] != p[0] or p0[1] != p[1]:
                if p0[1] == p[1]:
                    fill_rect(img, p0[0], p0[1] - half, p[0], p[1] + half, color)
                else:
                    fill_rect(img, p0[0] - half, p0[1], p[0] + half, p[1], color)
            fill_circle(img, p[0], p[1], (thickness + 1) >> 1, color)
        p0 = p


def clip_line(w, h, p1, p2):
    """cv::clipLine on a Size2l and two Point2l (Cohen-Sutherland, intercepts in double, truncated)."""
    right, bottom = w - 1, h - 1
    x1, y1 = p1
    x2, y2 = p2
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += int(float(a - y1) * float(x2 - x1) / float(y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += int(float(a - y2) * float(x2 - x1) / float(y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += int(float(a - x1) * float(y2 - y1) / float(x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += int(float(a - x2) * float(y2 - y1) / float(x2 - x1))
                x2 = a
                c2 = 0
    return (c1 | c2) == 0, (x1, y1), (x2, y2)


def line_aa_setup(w, h, pt1, pt2):
    """LineAA's set-up for a 16.16 segment: None when clipped away, else (x_major, start column/row, first minor
    coordinate in 16.16, step, number of steps - 1, ep_table)."""
    ok, pt1, pt2 = clip_line(w << XY_SHIFT, h << XY_SHIFT, pt1, pt2)
    if not ok:
        return None
    (x1, y1), (x2, y2) = pt1, pt2
    dx, dy = x2 - x1, y2 - y1
    ax, ay = abs(dx), abs(dy)
    if ax > ay:
        if dx < 0:                             # walk left to right
            x1, x2, y1, y2, dy = x2, x1, y2, y1, -dy
        step = tdiv(dy << XY_SHIFT, ax | 1)
        x2 += XY_ONE
        ecount = (x2 >> XY_SHIFT) - (x1 >> XY_SHIFT)
        j = -(x1 & (XY_ONE - 1))
        y1 += ((step * j) >> XY_SHIFT) + (XY_ONE >> 1)
        i, j = (x1 >> (XY_SHIFT - 7)) & 0x78, (x2 >> (XY_SHIFT - 7)) & 0x78
        start, minor = x1 >> XY_SHIFT, y1
    else:
        if dy < 0:
            x1, x2, y1, y2, dx = x2, x1, y2, y1, -dx
        step = tdiv(dx << XY_SHIFT, ay | 1)
        y2 += XY_ONE
        ecount = (y2 >> XY_SHIFT) - (y1 >> XY_SHIFT)
        j = -(y1 & (XY_ONE - 1))
        x1 += ((step * j) >> XY_SHIFT) + (XY_ONE >> 1)
        i, j = (y1 >> (XY_SHIFT - 7)) & 0x78, (y2 >> (XY_SHIFT - 7)) & 0x78
        start, minor = y1 >> XY_SHIFT, x1
    slope = (step >> (XY_SHIFT - 5)) & 0x3F
    slope ^= 0x3F if step < 0 else 0
    slope = 0x100 if slope & 0x20 else SLOPE_CORR[slope]
    t0 = slope << 7
    t1 = ((0x78 - i) | 4) * slope
    t2 = (j | 4) * slope
    ep = [0] * 9
    ep[8] = slope
    ep[1] = ep[3] = ((((j - i) & 0x78) | 4) * slope >> 8) & 0x1FF
    ep[2] = (t1 >> 8) & 0x1FF
    ep[4] = ((((j - i) + 0x80) | 4) * slope >> 8) & 0x1FF
    ep[5] = ((t1 + t0) >> 8) & 0x1FF
    ep[6] = (t2 >> 8) & 0x1FF
    ep[7] = ((t2 + t0) >> 8) & 0x1FF
    return ax > ay, start, minor, step, ecount, ep


def blend(img, x, y, color, a):
    """LineAA's put: OpenCV 4.13 applies the rounded step towards the colour twice for 3-channel images."""
    c = np.asarray(color, np.int64)
    px = img[y, x].astype(np.int64)
    px += ((c - px) * a + 127) >> 8
    px += ((c - px) * a + 127) >> 8
    img[y, x] = px


def line_aa(img, pt1, pt2, color):
    """LineAA: anti-aliased 1-pixel line between 16.16 points, blended into a 3-channel uint8 image."""
    h, w = img.shape[:2]
    s = line_aa_setup(w, h, pt1, pt2)
    if s is None:
        return
    x_major, start, minor, step, ecount, ep = s
    size_major, size_minor = (w, h) if x_major else (h, w)
    scount = 0
    major = start
    while ecount >= 0:
        if 0 <= major < size_major:
            m = (minor >> XY_SHIFT) - 1
            corr = ep[(((scount >= 2) + 1) & (scount | 2)) * 3 + (((ecount >= 2) + 1) & (ecount | 2))]
            dist = (minor >> (XY_SHIFT - 5)) & 31
            for k, f in enumerate((FILTER[dist + 32], FILTER[dist], FILTER[63 - dist])):
                if 0 <= m + k < size_minor:
                    a = (corr * f >> 8) & 0xFF
                    if x_major:
                        blend(img, major, m + k, color, a)
                    else:
                        blend(img, m + k, major, color, a)
        major += 1
        minor += step
        scount += 1
        ecount -= 1


def text_strokes(codes, org, scale):
    """putText's polylines as lists of 16.16 points, in drawing order (FONT_HERSHEY_SIMPLEX, bottomLeftOrigin=False).
    Strokes of one point are not drawn."""
    hscale = cv_round(scale * XY_ONE)
    view_x = org[0] << XY_SHIFT
    view_y = (org[1] << XY_SHIFT) - BASE_LINE * hscale
    strokes = []
    for c in codes:
        g = GLYPHS[c - 32]
        view_x -= (ord(g[0]) - 82) * hscale
        for stroke in g[2:].split(" "):
            pts = [((ord(stroke[k]) - 82) * hscale + view_x, (ord(stroke[k + 1]) - 82) * hscale + view_y)
                   for k in range(0, len(stroke), 2)]
            if len(pts) > 1:
                strokes.append(pts)
        view_x += (ord(g[1]) - 82) * hscale
    return strokes


def text_segments(codes, org, scale):
    return [seg for pts in text_strokes(codes, org, scale) for seg in zip(pts[:-1], pts[1:])]


def fill_convex_poly_aa(img, v, color):
    """FillConvexPoly(img, v, n, color, LINE_AA, XY_SHIFT): LineAA along every edge (from the last vertex round),
    then the scanline fill, opaque, rows ymin .. ymax with edges re-walked only while y < ymax or y == ymin."""
    h, w = img.shape[:2]
    n = len(v)
    delta = XY_ONE >> 1
    p0 = v[-1]
    for p in v:
        line_aa(img, p0, p, color)
        p0 = p
    xs_, ys_ = [p[0] for p in v], [p[1] for p in v]
    imin = min(range(n), key=lambda k: (ys_[k], k))
    xmin, xmax = (min(xs_) + delta) >> XY_SHIFT, (max(xs_) + delta) >> XY_SHIFT
    ymin, ymax = (min(ys_) + delta) >> XY_SHIFT, (max(ys_) + delta) >> XY_SHIFT
    if n < 3 or xmax < 0 or ymax < 0 or xmin >= w or ymin >= h:
        return
    ymax = min(ymax, h - 1)
    edges = n
    e = [dict(idx=imin, di=1, x=-XY_ONE, dx=0, ye=ymin), dict(idx=imin, di=n - 1, x=-XY_ONE, dx=0, ye=ymin)]
    y = ymin
    while True:
        if y < ymax or y == ymin:
            for E in e:
                if y >= E["ye"]:
                    idx0, di = E["idx"], E["di"]
                    idx = (idx0 + di) % n
                    while True:
                        edges -= 1
                        if edges < 0:
                            break
                        ty = (v[idx][1] + delta) >> XY_SHIFT
                        if ty > y:
                            xs, xe = v[idx0][0], v[idx][0]
                            E["ye"] = ty
                            E["dx"] = tdiv((xe - xs) * 2 + (ty - y), 2 * (ty - y))
                            E["x"] = xs
                            E["idx"] = idx
                            break
                        idx0 = idx
                        idx = (idx + di) % n
        if edges < 0:
            break
        if y >= 0:
            left, right = (1, 0) if e[0]["x"] > e[1]["x"] else (0, 1)
            x1 = (e[left]["x"] + XY_ONE - 1) >> XY_SHIFT
            x2 = e[right]["x"] >> XY_SHIFT
            x1, x2 = max(x1, 0), min(x2, w - 1)
            if x1 <= x2:                                   # ICV_HLINE draws nothing for x1 > x2
                img[y, x1:x2 + 1] = color
        e[0]["x"] += e[0]["dx"]
        e[1]["x"] += e[1]["dx"]
        y += 1
        if y > ymax:
            break


def cap_polygon(center, radius):
    """EllipseEx(center, (radius, radius), 0, 0, 360, filled)'s polygon: ellipse2Poly in double with OpenCV's float
    SinTable, each point rounded to 16.16 as EllipseEx does, repeats dropped."""
    r = (radius + (XY_ONE >> 1)) >> XY_SHIFT
    step = 90 if r < 3 else 30 if r < 10 else 18 if r < 15 else 5
    pts = []
    i = 0
    while i < 360 + step:
        a = min(i, 360)
        x = radius * SIN_TABLE[450 - a]
        y = radius * SIN_TABLE[a]
        pts.append((center[0] + x * 1.0 - y * 0.0, center[1] + x * 0.0 + y * 1.0))
        i += step
    out = []
    for px, py in pts:
        qx = cv_round(px / XY_ONE) << XY_SHIFT
        qy = cv_round(py / XY_ONE) << XY_SHIFT
        q = (qx + cv_round(px - qx), qy + cv_round(py - qy))
        if not out or out[-1] != q:
            out.append(q)
    if len(out) == 1:
        out = [tuple(center)] * 2
    return out


def thick_line_aa(img, p0, p1, color, thickness, flags):
    """ThickLine(p0, p1, thickness >= 2, LINE_AA, flags) on 16.16 points: the anti-aliased quad, then a round cap
    at p0 (flags & 1) and at p1 (flags & 2)."""
    dx = (p0[0] - p1[0]) / XY_ONE
    dy = (p1[1] - p0[1]) / XY_ONE
    r = dx * dx + dy * dy
    odd = thickness & 1
    half = thickness << (XY_SHIFT - 1)
    if abs(r) > 2.220446049250313e-16:
        r = (half + odd * XY_ONE * 0.5) / math.sqrt(r)
        ex, ey = cv_round(dy * r), cv_round(dx * r)
        fill_convex_poly_aa(img, [(p0[0] + ex, p0[1] + ey), (p0[0] - ex, p0[1] - ey), (p1[0] - ex, p1[1] - ey),
                                  (p1[0] + ex, p1[1] + ey)], color)
    for i, p in enumerate((p0, p1)):
        if flags & (i + 1):
            fill_convex_poly_aa(img, cap_polygon(p, half), color)


def put_text(img, codes, org, scale, color, thickness):
    """cv2.putText(img, text, org, FONT_HERSHEY_SIMPLEX, scale, color, thickness, LINE_AA)."""
    for pts in text_strokes(codes, org, scale):
        for k in range(1, len(pts)):
            if thickness <= 1:
                line_aa(img, pts[k - 1], pts[k], color)
            else:
                thick_line_aa(img, pts[k - 1], pts[k], color, thickness, 3 if k == 1 else 2)


def plot_one_box(img, coord, label=None, color=None, line_thickness=None):
    """The reference's plot_one_box with every cv2 call restated (color must be given)."""
    tl = line_thickness or int(round(0.002 * max(img.shape[0:2])))
    c1, c2 = (int(coord[0]), int(coord[1])), (int(coord[2]), int(coord[3]))
    rectangle(img, c1, c2, color, tl)
    if label:
        codes = text_codes(label)
        _, c2, org, tf = label_layout(codes, tl, c1)
        rectangle(img, c1, c2, color, -1)
        put_text(img, codes, org, float(tl) / 3, (0, 0, 0), tf)


def score_text(score):
    """The reference's label suffix for a float32 score."""
    return ", {:.2f}%".format(np.float32(score) * 100)


def draw_detections(img, boxes, scores, labels, class_names, color_table, line_thickness=None):
    """test_single_image.py's loop over one image's detections, in order."""
    for b, s, l in zip(boxes, scores, labels):
        plot_one_box(img, b, label=class_names[l] + score_text(s), color=color_table[l],
                     line_thickness=line_thickness)
    return img
