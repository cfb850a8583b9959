"""Fixtures of the device JPEG encoder (tests/golden/jpeg_enc.npz), from OpenCV's own encoder.

Run with OpenCV 4.13 (libjpeg-turbo 3.1): `python tests/golden/make_golden_jpeg_enc.py`.  Each case is an input
(tests/jpeg_enc_cases.py rebuilds it from a seed: noise, gradient, flat or a crop of dog.jpg / messi.jpg, BGR or grey)
and encoder arguments; it stores cv2.imencode's file, in full up to 4096 bytes and as SHA-256 and length above, and
the SHA-256 of cv2.imdecode of that file (IMREAD_COLOR), for the decode round trip.  Covered: sizes 1 x 1 to
500 x 375 and edge shapes that are no MCU multiple, every sampling mode and grey, qualities 0-101, luma / chroma
pairs, restart intervals 0, 1, 3 and 7, and dog.jpg and messi.jpg whole."""
import hashlib
import json
import os
import re
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import jpeg_enc_cases as E  # noqa: E402
from tests import jpeg_enc_ref as R  # noqa: E402

SIZES = [(1, 1), (7, 9), (15, 16), (16, 15), (17, 33), (33, 1), (1, 33), (375, 500), (500, 375)]
MODES = ["411", "420", "422", "440", "444", "grey"]
KINDS = ["noise", "gradient", "flat", "dog.jpg"]
QUALITIES = [0, 1, 10, 50, 75, 90, 95, 100, 101]
RESTARTS = [0, 1, 3, 7]


def cases():
    out, seed = [], 1000
    for si, (h, w) in enumerate(SIZES):
        for mi, mode in enumerate(MODES):
            seed += 1
            out.append(dict(h=h, w=w, kind=KINDS[(si + mi) % 4], grey=mode == "grey", seed=seed,
                            kw=dict(quality=QUALITIES[(si * 6 + mi) % 9], sampling="420" if mode == "grey" else mode,
                                    restart_interval=RESTARTS[(si + 2 * mi) % 4])))
    for q in QUALITIES:
        for mode in ("420", "grey"):
            seed += 1
            out.append(dict(h=40, w=56, kind="dog.jpg", grey=mode == "grey", seed=seed,
                            kw=dict(quality=q, sampling="420", restart_interval=0)))
    for lq, cq in [(90, 50), (50, 90), (75, 75), (100, 0), (30, None)]:
        for mode in ("420", "411"):
            seed += 1
            kw = dict(quality=95, sampling=mode, restart_interval=0, luma_quality=lq)
            if cq is not None:
                kw["chroma_quality"] = cq
            out.append(dict(h=33, w=47, kind="messi.jpg", grey=False, seed=seed, kw=kw))
    seed += 1
    out.append(dict(h=33, w=47, kind="messi.jpg", grey=False, seed=seed, kw=dict(quality=80, chroma_quality=20)))
    for ri in RESTARTS:
        seed += 1
        out.append(dict(h=375, w=500, kind="dog.jpg", grey=False, seed=seed, kw=dict(quality=95, restart_interval=ri)))
    for name, shape in (("dog.jpg", (576, 768)), ("messi.jpg", (729, 1296))):
        for kw in (dict(quality=95), dict(quality=75), dict(quality=90, sampling="444", restart_interval=3)):
            seed += 1
            out.append(dict(h=shape[0], w=shape[1], kind=name, grey=False, seed=seed, kw=kw, whole=True))
    return out


def main():
    turbo = re.search(r"libjpeg-turbo \(ver ([\d.]+)", cv2.getBuildInformation())
    meta = {"opencv": cv2.__version__, "libjpeg_turbo": turbo.group(1) if turbo else "", "cases": []}
    arrays = {}
    for k, c in enumerate(cases()):
        img = E.image(c)
        data = cv2.imencode(".jpg", img, R.cv2_params(**c["kw"]))[1].tobytes()
        c["name"] = f"{c['kind']}_{c['h']}x{c['w']}_{'grey' if c['grey'] else c['kw'].get('sampling', '420')}_{k}"
        c["length"] = len(data)
        c["sha256"] = hashlib.sha256(data).hexdigest()
        if len(data) <= 4096:
            arrays[f"jpg_{k}"] = np.frombuffer(data, np.uint8)
        back = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)
        c["roundtrip_sha256"] = hashlib.sha256(np.ascontiguousarray(back).tobytes()).hexdigest()
        meta["cases"].append(c)
    arrays["meta"] = np.frombuffer(json.dumps(meta).encode(), np.uint8)
    np.savez_compressed(os.path.join(HERE, "jpeg_enc.npz"), **arrays)
    print(len(meta["cases"]), "cases,", os.path.getsize(os.path.join(HERE, "jpeg_enc.npz")), "bytes")


if __name__ == "__main__":
    main()
