"""Seeded drawing cases for the plot tests: an image and a list of plot_one_box calls, rebuilt from the seed.

Coverage: tl 0..6 from the image size (including the round-half-even tie at 250 px: 0.002 * 250 = 0.5 -> 0, and
long sides of 1250 px and more, whose labels have thick strokes) and explicit thicknesses 1..12; boxes inside,
straddling each edge, fully outside (up to 4x the image size), degenerate, swapped and with negative fractional coordinates; every printable ASCII character, COCO
names, empty / None labels and non-ASCII names; several overlapping boxes, so order matters."""
import os
import string

import numpy as np

COCO = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolov3_tensorflow_b200", "data",
                         "coco.names")).read().split("\n")[:80]
ASCII = string.printable[:95]                             # ' ' .. '~' in some order, plus nothing else
NAMES = COCO + ["", "é", "日本", "ß?x", "naïve café", "\t", ASCII[:40], ASCII[40:]]


def case(seed):
    """-> (image uint8 [h, w, 3], [(coord float32 [4], label or None, color, line_thickness or None)], score list)"""
    r = np.random.default_rng(seed)
    kind = seed % 5
    if kind == 4:
        h, w = int(r.integers(30, 240)), int(r.integers(1250, 3250))    # tl 3..6: thick anti-aliased text
    elif kind == 0:
        h, w = int(r.integers(8, 250)), int(r.integers(8, 250))          # tl 0
    elif kind == 1:
        h, w = int(r.integers(250, 750)), int(r.integers(100, 750))      # tl 0 (250), 1
    elif kind == 2:
        h, w = int(r.integers(100, 400)), int(r.integers(751, 1249))     # tl 2
    else:
        h, w = int(r.integers(30, 600)), int(r.integers(30, 600))
    if seed % 17 == 0:
        h, w = 250, int(r.integers(30, 250))                            # 0.5 rounds to 0
    img = r.integers(0, 256, (h, w, 3), dtype=np.uint8)
    calls = []
    for _ in range(int(r.integers(1, 6))):
        span = 4.0 if r.random() < 0.3 else 1.3
        x = r.uniform(-span * w, span * w, 2)
        y = r.uniform(-span * h, span * h, 2)
        if r.random() < 0.15:
            x[1] = x[0]                                                  # degenerate
        if r.random() < 0.15:
            y[1] = y[0]
        if r.random() < 0.3:                                             # mostly a box near the image
            x = np.sort(r.uniform(-0.2 * w, 1.2 * w, 2))
            y = np.sort(r.uniform(-0.2 * h, 1.2 * h, 2))
        coord = np.array([x[0], y[0], x[1], y[1]], np.float32)
        color = [int(v) for v in r.integers(0, 256, 3)]
        lt = None
        label = None
        u = r.random()
        if kind == 3 and u < 0.3:
            lt = int(r.integers(1, 13))                                  # explicit thickness
        if r.random() < 0.85:
            label = NAMES[int(r.integers(0, len(NAMES)))]
            if r.random() < 0.7:
                label += ", {:.2f}%".format(np.float32(r.random()) * 100)
        calls.append((coord, label, color, lt))
    return img, calls
