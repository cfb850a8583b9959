"""Fixtures of the device JPEG decoder (tests/golden/jpeg.npz), from OpenCV's own encoder and decoder.

Run with OpenCV 4.13 (libjpeg-turbo 3.1) and Pillow: `python tests/golden/make_golden_jpeg.py`.  It writes
  * synthetic cv2.imencode files: sizes 1x1 .. 500x375, 4:4:4 / 4:2:2 / 4:4:0 / 4:2:0 and grey, qualities 10-100,
    restart intervals 0, 1, 3 and odd, IMWRITE_JPEG_OPTIMIZE tables; natural crops of the demo images, noise, flat
    and gradient content.  Expected output cv2.imdecode(..., IMREAD_COLOR), in full up to 64 x 64 pixels, as a
    SHA-256 above;
  * EXIF orientations 1-8 (an APP1 segment injected after SOI, little- and big-endian TIFF);
  * rejected files with the expected reason (progressive, 4:1:1, CMYK from Pillow) and corrupt files (truncated,
    bit-flipped) with the expected status of tests/jpeg_ref.py;
  * SHA-256 and shape of cv2.imread of dog.jpg and messi.jpg (copied next to this file from the reference's
    data/demo_data)."""
import hashlib
import io
import json
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import jpeg_ref as R  # noqa: E402

SAMP = {"444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
        "440": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440, "420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420}


def content(kind, h, w, rng, demo):
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "flat":
        return np.full((h, w, 3), rng.integers(0, 256, 3), np.uint8)
    if kind == "gradient":
        g = np.add.outer(np.arange(h) * 255 // max(h, 1), np.arange(w) * 255 // max(w, 1))
        return np.clip(g[:, :, None] // 2 + np.array([0, 40, 90]), 0, 255).astype(np.uint8)
    d = demo[rng.integers(0, len(demo))]
    y0, x0 = rng.integers(0, d.shape[0] - h + 1), rng.integers(0, d.shape[1] - w + 1)
    return d[y0:y0 + h, x0:x0 + w].copy()


def encode(img, q, samp, ri, opt):
    ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMP[samp],
                                         cv2.IMWRITE_JPEG_RST_INTERVAL, ri, cv2.IMWRITE_JPEG_OPTIMIZE, opt])
    assert ok
    return enc.tobytes()


def with_orientation(jpg, o, big_endian):
    e = ">" if big_endian else "<"
    tiff = (b"MM" if big_endian else b"II") + np.array([42], e + "u2").tobytes() + np.array([8], e + "u4").tobytes()
    tiff += np.array([1], e + "u2").tobytes() + np.array([0x0112, 3], e + "u2").tobytes()
    tiff += np.array([1], e + "u4").tobytes() + np.array([o, 0], e + "u2").tobytes() + b"\0\0\0\0"
    seg = b"Exif\0\0" + tiff
    return jpg[:2] + b"\xff\xe1" + (len(seg) + 2).to_bytes(2, "big") + seg + jpg[2:]


def main():
    rng = np.random.default_rng(2026)
    demo = [cv2.imread(os.path.join(HERE, n)) for n in ("dog.jpg", "messi.jpg")]
    out, meta = {}, {"opencv": cv2.__version__, "cases": []}

    def add(name, jpg, note, expect=None, status=0, reason=None):
        k = len(meta["cases"])
        out[f"jpg_{k}"] = np.frombuffer(jpg, np.uint8)
        case = dict(name=name, note=note, status=status, reason=reason)
        if expect is not None:
            case["shape"] = list(expect.shape)
            case["sha256"] = hashlib.sha256(expect.tobytes()).hexdigest()
            if expect.shape[0] * expect.shape[1] <= 64 * 64:
                out[f"exp_{k}"] = expect
        meta["cases"].append(case)

    sizes = [(1, 1), (7, 5), (8, 8), (9, 17), (16, 16), (33, 47), (127, 255), (375, 500), (500, 375)]
    kinds = ["natural", "noise", "flat", "gradient"]
    for si, (h, w) in enumerate(sizes):
        for pi, samp in enumerate(list(SAMP) + ["grey"]):
            kind = kinds[(si + pi) % 4] if h * w > 1 else "flat"
            if kind == "noise" and h * w > 64 * 64:   # keeps the file small; noise stays covered below 64 x 64
                kind = "natural"
            img = content(kind, h, w, rng, demo)
            q = int(rng.choice([10, 30, 50, 75, 90, 95, 100]))
            ri = int(rng.choice([0, 1, 3, 5]))
            opt = int(rng.random() < 0.3)
            src = img[:, :, 0].copy() if samp == "grey" else img
            jpg = encode(src, q, "444" if samp == "grey" else samp, ri, opt)
            exp = cv2.imdecode(np.frombuffer(jpg, np.uint8), cv2.IMREAD_COLOR)
            add(f"{h}x{w}_{samp}_{kind}_q{q}_ri{ri}_opt{opt}", jpg, "synthetic", exp)
    # VOC-size photographs: crops of the demo images, q95 4:2:0 as VOC's own files, with and without restart intervals
    for h, w in ((375, 500), (500, 375)):
        for ri in (0, 4):
            jpg = encode(content("natural", h, w, rng, demo), 95, "420", ri, 0)
            add(f"voc_{h}x{w}_ri{ri}", jpg, "synthetic", cv2.imdecode(np.frombuffer(jpg, np.uint8), 1))
    for samp in SAMP:   # noise at quality 100: IDCT outputs at the clamp
        img = content("noise", 24, 40, rng, demo)
        jpg = encode(img, 100, samp, 0, 0)
        add(f"24x40_{samp}_noise_q100", jpg, "synthetic", cv2.imdecode(np.frombuffer(jpg, np.uint8), 1))
    base = encode(content("natural", 33, 47, rng, demo), 90, "420", 2, 0)
    for o in range(1, 9):
        jpg = with_orientation(base, o, big_endian=o % 2 == 0)
        exp = cv2.imdecode(np.frombuffer(jpg, np.uint8), cv2.IMREAD_COLOR)
        assert np.array_equal(exp, np.ascontiguousarray(R.orient(cv2.imdecode(np.frombuffer(base, np.uint8), 1), o)))
        add(f"exif_{o}", jpg, "orientation", exp)
    img = content("natural", 48, 64, rng, demo)
    ok, prog = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
    add("progressive", prog.tobytes(), "rejected", reason="progressive JPEG")
    ok, s411 = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411])
    add("411", s411.tobytes(), "rejected", reason="sampling factors")
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(img[:, :, ::-1]).convert("CMYK").save(buf, "JPEG", quality=90)
    add("cmyk", buf.getvalue(), "rejected", reason="4 components")
    meta["pillow"] = Image.__version__ if hasattr(Image, "__version__") else ""
    # SOS listing the components in another order than SOF (libjpeg accepts it; rejected here)
    b = bytearray(encode(content("natural", 16, 16, rng, demo), 90, "444", 0, 0))
    sos = R.parse(bytes(b))["scan_start"] - 10            # 3 components: 12-byte segment body, ids at +1, +3, +5
    b[sos + 1:sos + 3], b[sos + 3:sos + 5] = b[sos + 3:sos + 5], b[sos + 1:sos + 3]
    add("sos_order", bytes(b), "rejected", reason="another order than SOF")

    def corrupt(name, b):
        """A damaged file: its status (tests/jpeg_ref.py) if nonzero; otherwise the restatement's image, which must
        be cv2's, or a recorded divergence where libjpeg's recovery differs."""
        img2, st = R.decode(b)
        if st:
            add(name, b, "corrupt", status=int(st))
            return int(st)
        exp = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
        if exp is not None and np.array_equal(exp, img2):
            add(name, b, "synthetic", exp)
        else:
            meta["divergent"].append(name)
            add(name, b, "divergent", img2)
        return 0

    meta["divergent"] = []
    for name, ri in (("corrupt_base", 0), ("corrupt_base_ri", 4)):
        jpg = encode(content("natural", 64, 96, rng, demo), 85, "420", ri, 0)
        add(name, jpg, "synthetic", cv2.imdecode(np.frombuffer(jpg, np.uint8), 1))
        start = R.parse(jpg)["scan_start"]
        ln = len(jpg) - start
        for frac in (0.3, 0.7, 0.97):
            corrupt(f"{name}_trunc{frac}", jpg[:start + int(ln * frac)])
        for k in range(12):
            b = bytearray(jpg)
            b[start + int(rng.integers(0, ln - 2))] ^= 1 << int(rng.integers(0, 8))
            corrupt(f"{name}_flip{k}", bytes(b))
        q = start + ln // 4
        corrupt(f"{name}_marker", jpg[:q] + b"\xff\xe0" + jpg[q:])             # APP0 inside the entropy data
        corrupt(f"{name}_ffff", jpg[:q] + b"\xff\x00" * 4 + jpg[q:])           # 32 one-bits: no table holds them
        if ri:
            rst = [i for i in range(start, len(jpg) - 1) if jpg[i] == 0xFF and 0xD0 <= jpg[i + 1] <= 0xD7]
            b = bytearray(jpg)
            b[rst[1] + 1] = 0xD0 + (b[rst[1] + 1] - 0xD0 + 3) % 8
            corrupt(f"{name}_rst_order", bytes(b))
            corrupt(f"{name}_rst_extra", jpg[:-2] + bytes([0xFF, 0xD0 + len(rst) % 8]) + jpg[-2:])
        found = False   # random bytes over a stretch of the scan, until one decodes a coefficient past k = 63
        for k in range(400):
            b = bytearray(jpg)
            p0 = start + int(rng.integers(0, ln // 2))
            b[p0:p0 + 6] = bytes(rng.integers(0, 255, 6, dtype=np.uint8))
            _, st = R.decode(bytes(b))
            if st & R.BAD_INDEX:
                corrupt(f"{name}_index", bytes(b))
                found = True
                break
        assert found
    bits = 0
    for c in meta["cases"]:
        bits |= c["status"]
    assert bits == 31, f"the corrupt fixtures cover status bits {bits:#x}, not all five"
    print("flips whose restatement output differs from cv2.imdecode:", meta["divergent"])
    for n in ("dog.jpg", "messi.jpg"):
        im = cv2.imread(os.path.join(HERE, n))
        meta[n] = dict(shape=list(im.shape), sha256=hashlib.sha256(im.tobytes()).hexdigest(),
                       file_sha256=hashlib.sha256(open(os.path.join(HERE, n), "rb").read()).hexdigest())
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), np.uint8)
    np.savez_compressed(os.path.join(HERE, "jpeg.npz"), **out)
    print(len(meta["cases"]), "cases,", os.path.getsize(os.path.join(HERE, "jpeg.npz")), "bytes")


if __name__ == "__main__":
    main()
