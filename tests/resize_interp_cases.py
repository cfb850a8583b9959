"""Seeded cases of the training resize tests (cv2.resize with INTER_CUBIC, INTER_AREA, INTER_LANCZOS4): the source
images are rebuilt from the seed, so the goldens store only what the reference made of them.

SMALL (results stored in full): 1 x 1, 1 x N and N x 1 sources, odd sizes, same size in and out, exact 2x, 3x and 4x
downscales, non-integer downscales, pure upscales and both mixed-axis cases (one axis shrinks, the other grows).
LARGE (results stored as SHA-256): a 4x-expanded crop wider than 2000 px down to 320, and training-like crops to every
multi-scale target 320..608 in steps of 32.  Each case runs letterboxed and stretched."""
import numpy as np

INTERPS = (2, 3, 4)

# src h, src w, new w, new h
SMALL = [(1, 1, 32, 24), (1, 17, 24, 16), (19, 1, 16, 24), (33, 61, 48, 40), (41, 23, 37, 53), (48, 64, 64, 48),
         (64, 96, 48, 32), (63, 93, 31, 21), (64, 96, 24, 16), (100, 75, 40, 32), (30, 40, 97, 73), (40, 90, 60, 100),
         (90, 40, 100, 60), (7, 5, 9, 3), (99, 123, 45, 37), (16, 16, 16, 16), (5, 300, 64, 64)]
LARGE = [(1517, 2013, 320, 320), (2203, 1650, 320, 320)] + [
    (int(h), int(w), s, s) for (h, w), s in zip(((375, 500), (500, 375), (281, 437), (611, 301), (333, 500),
                                                   (120, 97), (480, 640), (457, 611), (701, 1003), (608, 608)),
                                                  range(320, 609, 32))]


def source(i, shape):
    """Case i's uint8 BGR source of (h, w)."""
    return np.random.default_rng(9000 + i).integers(0, 256, (shape[0], shape[1], 3), dtype=np.uint8)


def boxes(i, h, w, v=4):
    """Case i's ground truth as parse_data holds it: float32 [v, 5] with the mix-up weight column."""
    r = np.random.default_rng(19000 + i)
    x0, x1, y0, y1 = r.uniform(0, w, v), r.uniform(0, w, v), r.uniform(0, h, v), r.uniform(0, h, v)
    return np.stack([np.minimum(x0, x1), np.minimum(y0, y1), np.maximum(x0, x1), np.maximum(y0, y1), np.ones(v)],
                    1).astype(np.float32)


def cases():
    """-> [(index, (src h, src w, new w, new h), stored in full)]"""
    return [(i, c, i < len(SMALL)) for i, c in enumerate(SMALL + LARGE)]
