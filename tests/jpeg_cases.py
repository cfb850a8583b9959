"""The fixtures of tests/golden/jpeg.npz (written by tests/golden/make_golden_jpeg.py), for the JPEG tests."""
import hashlib
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load():
    z = np.load(os.path.join(GOLDEN, "jpeg.npz"))
    meta = json.loads(bytes(z["meta"]).decode())
    cases = []
    for k, c in enumerate(meta["cases"]):
        c = dict(c, data=z[f"jpg_{k}"].tobytes())
        if f"exp_{k}" in z:
            c["expect"] = z[f"exp_{k}"]
        cases.append(c)
    return meta, cases


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def demo(name):
    with open(os.path.join(GOLDEN, name), "rb") as f:
        return f.read()
