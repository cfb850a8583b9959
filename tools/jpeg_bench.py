"""Device JPEG decode vs cv2.imdecode at batch 64, from committed fixtures only (tests/golden).

  python tools/jpeg_bench.py [--batch 64] [--iters 20]

Reports the card and its power limit, device decode images/s and compressed MB/s for the VOC-size photographs
(q95 4:2:0 crops of the demo images, 375 x 500 and 500 x 375, with and without restart intervals) and messi.jpg, cv2.imdecode on one host core and on all host
cores (a thread pool) where cv2 imports, and end to end bytes -> decode_jpeg_batch -> preprocess_batch -> detect_raw
against host decode -> preprocess_batch -> detect_raw.  Exits nonzero if any decoded image differs from its golden
or, where cv2 imports, from cv2.imdecode."""
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
from tests.jpeg_cases import load, sha, demo  # noqa: E402
from yolov3_tensorflow_b200.utils.data_aug import decode_jpeg_batch, preprocess_batch  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "jpeg_bench needs a GPU"
    meta, cases = load()
    try:
        import cv2
    except ImportError:
        cv2 = None
    voc = [c for c in cases if c["name"].startswith("voc_")]   # q95 4:2:0 photographs, 375 x 500 and 500 x 375
    sets = {"voc_restart": [c for c in voc if not c["name"].endswith("_ri0")],
            "voc_no_restart": [c for c in voc if c["name"].endswith("_ri0")],
            "messi": [dict(data=demo("messi.jpg"), sha256=meta["messi.jpg"]["sha256"])]}
    res = {"card": card(), "batch": a.batch, "host_cores": os.cpu_count(), "sets": {}}
    ok = True
    for name, pool in sets.items():
        if not pool:
            continue
        files = [pool[i % len(pool)]["data"] for i in range(a.batch)]
        want = [pool[i % len(pool)]["sha256"] for i in range(a.batch)]
        p = decode_jpeg_batch(files)
        for i in range(a.batch):
            got = p.image(i).cpu().numpy()
            if sha(got) != want[i]:
                ok = False
            if cv2 is not None and not np.array_equal(got, cv2.imdecode(np.frombuffer(files[i], np.uint8), 1)):
                ok = False
        mb = sum(len(f) for f in files) / 1e6
        t = timed(lambda: decode_jpeg_batch(files, check=False), a.iters)
        r = {"device_img_s": a.batch / t, "device_MB_s": mb / t, "device_ms": t * 1e3, "compressed_MB": mb}
        if cv2 is not None:
            dec = lambda f: cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)  # noqa: E731
            t0 = time.perf_counter()
            for f in files:
                dec(f)
            r["cv2_1core_img_s"] = a.batch / (time.perf_counter() - t0)
            with ThreadPoolExecutor(os.cpu_count()) as ex:
                list(ex.map(dec, files))
                t0 = time.perf_counter()
                for _ in range(3):
                    list(ex.map(dec, files))
                r["cv2_allcores_img_s"] = 3 * a.batch / (time.perf_counter() - t0)
        res["sets"][name] = r
    if cv2 is not None and sets["voc_restart"]:
        import yolov3_tensorflow_b200 as pkg
        from oracle import yolov3_oracle as O
        m = pkg.yolov3(80, O.COCO_ANCHORS, dtype="fp16")
        m.set_params(O.make_params(80, seed=3, random_bn=True, det_scale=8.0, conf_bias=-2.0), "HWIO")
        files = [voc[i % len(voc)]["data"] for i in range(a.batch)]   # both VOC sets
        dev = lambda: m.detect_raw(preprocess_batch(decode_jpeg_batch(files, check=False), 416, 416)[0])  # noqa: E731
        host = lambda: m.detect_raw(preprocess_batch([cv2.imdecode(np.frombuffer(f, np.uint8), 1) for f in files],  # noqa: E731
                                                     416, 416)[0])
        res["end_to_end_img_s"] = {"device_decode": a.batch / timed(dev, a.iters),
                                   "host_decode_1core": a.batch / timed(host, max(2, a.iters // 4))}
    res["bytes_match"] = ok
    print(json.dumps(res))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
