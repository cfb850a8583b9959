"""Device JPEG encode vs cv2.imencode at batch 64, from committed fixtures only (tests/golden).

  python tools/jpeg_encode_bench.py [--batch 64] [--iters 20]

Inputs: the VOC-size photographs of tools/jpeg_bench.py (q95 4:2:0 files, 375 x 500 and 500 x 375), decoded on the
device first, and messi.jpg.  Each is encoded at q95 4:2:0 and at q75.  Reports the card and its power limit, device
images/s and output MB/s (CUDA events) for the device tensors alone (to_host=False) and for host bytes, cv2.imencode
on one host core and on all host cores (a thread pool) where cv2 imports, and decode -> encode end to end.  Exits
nonzero if any file differs from cv2.imencode (where cv2 imports) or from its golden."""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import jpeg_cases, jpeg_enc_cases  # noqa: E402
from yolov3_tensorflow_b200.utils.data_aug import decode_jpeg_batch, encode_jpeg_batch  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def timed(fn, iters):
    """Seconds per call by CUDA events around iters calls, after one warm-up call."""
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "jpeg_encode_bench needs a GPU"
    try:
        import cv2
    except ImportError:
        cv2 = None
    _, dec_cases = jpeg_cases.load()
    voc = [c["data"] for c in dec_cases if c["name"].startswith("voc_")]
    with open(os.path.join(jpeg_enc_cases.GOLDEN, "messi.jpg"), "rb") as f:
        messi = f.read()
    _, enc_cases = jpeg_enc_cases.load()
    golden = {(c["kind"], c["kw"].get("quality")): c for c in enc_cases
              if c.get("whole") and c["kw"].get("sampling", "420") == "420"}
    res = {"card": card(), "batch": a.batch, "host_cores": os.cpu_count(), "sets": {}}
    ok = True
    for name, pool in (("voc", voc), ("messi", [messi])):
        files = [pool[i % len(pool)] for i in range(a.batch)]
        packed = decode_jpeg_batch(files)
        host_imgs = [packed.image(i).cpu().numpy() for i in range(a.batch)]
        for q in (95, 75):
            kw = dict(quality=q, sampling="420")
            out = encode_jpeg_batch(packed, **kw)
            if name == "messi" and not jpeg_enc_cases.matches(golden[("messi.jpg", q)], out[0]):
                ok = False
            if cv2 is not None:
                prm = [cv2.IMWRITE_JPEG_QUALITY, q]
                ok &= all(o == cv2.imencode(".jpg", im, prm)[1].tobytes() for o, im in zip(out, host_imgs))
            mb = sum(len(o) for o in out) / 1e6
            t_dev = timed(lambda: encode_jpeg_batch(packed, to_host=False, **kw), a.iters)
            t_host = timed(lambda: encode_jpeg_batch(packed, **kw), a.iters)
            t_e2e = timed(lambda: encode_jpeg_batch(decode_jpeg_batch(files, check=False), **kw), a.iters)
            r = {"device_img_s": a.batch / t_dev, "device_MB_s": mb / t_dev, "device_ms": t_dev * 1e3,
                 "host_bytes_img_s": a.batch / t_host, "host_bytes_MB_s": mb / t_host,
                 "decode_encode_img_s": a.batch / t_e2e, "output_MB": mb}
            if cv2 is not None:
                enc = lambda im: cv2.imencode(".jpg", im, prm)  # noqa: E731
                t0 = time.perf_counter()
                for im in host_imgs:
                    enc(im)
                r["cv2_1core_img_s"] = a.batch / (time.perf_counter() - t0)
                with ThreadPoolExecutor(os.cpu_count()) as ex:
                    list(ex.map(enc, host_imgs))
                    t0 = time.perf_counter()
                    for _ in range(3):
                        list(ex.map(enc, host_imgs))
                    r["cv2_allcores_img_s"] = 3 * a.batch / (time.perf_counter() - t0)
            res["sets"][f"{name}_q{q}"] = r
    res["bytes_match"] = bool(ok)
    print(json.dumps(res))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
