"""The fixtures of tests/golden/jpeg_enc.npz (written by tests/golden/make_golden_jpeg_enc.py), for the JPEG encoder
tests.  Each case's input is rebuilt from its seed, or cropped from a demo image decoded by tests/jpeg_ref.py (which
equals cv2.imread), so the fixture stores only the expected files."""
import functools
import hashlib
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@functools.lru_cache(maxsize=None)
def demo(name):
    """cv2.imread of a demo image (tests/golden/<name>), without OpenCV."""
    from tests import jpeg_ref
    with open(os.path.join(GOLDEN, name), "rb") as f:
        return jpeg_ref.decode(f.read())[0]


def image(case):
    """The input image of a case: uint8 [H, W, 3] BGR, or [H, W] grey."""
    h, w, kind = case["h"], case["w"], case["kind"]
    rng = np.random.default_rng(case["seed"])
    if kind == "noise":
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    elif kind == "flat":
        img = np.full((h, w, 3), rng.integers(0, 256, 3), np.uint8)
    elif kind == "gradient":
        g = np.add.outer(np.arange(h) * 255 // max(h, 1), np.arange(w) * 255 // max(w, 1))
        img = np.clip(g[:, :, None] // 2 + np.array([0, 40, 90]), 0, 255).astype(np.uint8)
    else:                                  # a crop (or all) of a demo image
        d = demo(kind)
        y0, x0 = int(rng.integers(0, d.shape[0] - h + 1)), int(rng.integers(0, d.shape[1] - w + 1))
        img = d[y0:y0 + h, x0:x0 + w]
    img = np.ascontiguousarray(img)
    return np.ascontiguousarray(img[:, :, 1]) if case["grey"] else img


def load():
    z = np.load(os.path.join(GOLDEN, "jpeg_enc.npz"))
    meta = json.loads(bytes(z["meta"]).decode())
    cases = []
    for k, c in enumerate(meta["cases"]):
        c = dict(c)
        if f"jpg_{k}" in z:
            c["data"] = z[f"jpg_{k}"].tobytes()
        cases.append(c)
    return meta, cases


def sha(b):
    return hashlib.sha256(bytes(b) if not isinstance(b, np.ndarray) else np.ascontiguousarray(b).tobytes()).hexdigest()


def matches(case, data):
    """Whether encoder output `data` (bytes) is the case's expected file."""
    if "data" in case:
        return data == case["data"]
    return len(data) == case["length"] and sha(data) == case["sha256"]
