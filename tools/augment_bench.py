"""Training augmentation before the resize (parse_data(mode='train') up to the crop) for a batch of 375 x 500 images,
half of them mixed up as get_batch_data pairs them: the device path (utils.data_aug.augment_train_batch: host draws,
one parameter copy, one yb_augment_batch launch) against the reference-equivalent host chain (cv2.cvtColor + numpy,
one process per host core).  Prints one JSON line per batch size with images/s of both paths,
one launch's time (parameter copy + kernel) and its share of the HBM bound (source bytes read + output bytes written over 3.35 TB/s), and the card's name and power
limit read in the same run.  Usage: python tools/augment_bench.py [--batches 32 64] [--iters 20]"""
import argparse
import json
import os
import random
import subprocess
import sys
import time
from multiprocessing import Pool

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def _pairs(n, rng_np, rng_py):
    """get_batch_data's mix-up pairing (utils/data_utils.py:203-211)."""
    out = []
    for i in range(n):
        out.append(rng_py.choice([j for j in range(n) if j != i]) if rng_np.uniform(0, 1) < 0.5 else None)
    return out


def _host_chain(args):
    """One image through the reference's pre-resize chain with cv2 and numpy, drawing like it does."""
    import cv2
    img1, img2, boxes, seed = args
    np.random.seed(seed)
    random.seed(seed)
    from yolov3_tensorflow_b200.utils.data_aug import _draw_color, _draw_expand, _draw_mix, \
        random_crop_with_constraints
    if img2 is not None:
        r = _draw_mix()
        h, w = max(img1.shape[0], img2.shape[0]), max(img1.shape[1], img2.shape[1])
        mix = np.zeros((h, w, 3), np.float32)
        mix[:img1.shape[0], :img1.shape[1]] = img1.astype(np.float32) * r
        mix[:img2.shape[0], :img2.shape[1]] += img2.astype(np.float32) * (1. - r)
        img = mix.astype(np.uint8)
    else:
        img = img1
    bright, hue, sat, val = _draw_color()
    img = np.clip(img.astype(np.float32) + bright, 0, 255).astype(np.uint8)
    hsv = cv2.cvtColor(img, cv2.COLOR_BGR2HSV).astype(np.float32)
    hsv[..., 0] = (hsv[..., 0] + hue) % 180
    hsv[..., 1] *= sat
    hsv[..., 2] *= val
    img = cv2.cvtColor(np.clip(hsv, 0, 255).astype(np.uint8), cv2.COLOR_HSV2BGR)
    if np.random.uniform(0, 1) > 0.5:
        oh, ow, oy, ox = _draw_expand(*img.shape[:2])
        canvas = np.zeros((oh, ow, 3), np.uint8)
        canvas[oy: oy + img.shape[0], ox: ox + img.shape[1]] = img
        img = canvas
        boxes = boxes + np.array([ox, oy, ox, oy, 0], np.float32)
    boxes, (x0, y0, w, h) = random_crop_with_constraints(boxes, (img.shape[1], img.shape[0]))
    return np.ascontiguousarray(img[y0: y0 + h, x0: x0 + w]).nbytes


def _hbm_bytes(desc, params):
    """Bytes the kernel must move: the source pixels under each crop window (both images under a mix-up) plus the
    output."""
    total = 0
    for p in params:
        total += 3 * p.out_h * p.out_w
        for src in (p.src1, p.src2):
            if src < 0:
                continue
            h, w = int(desc[src, 1]), int(desc[src, 2])
            ix = max(0, min(p.crop_x + p.out_w, p.off_x + w) - max(p.crop_x, p.off_x))
            iy = max(0, min(p.crop_y + p.out_h, p.off_y + h) - max(p.crop_y, p.off_y))
            total += 3 * ix * iy
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import torch
    from yolov3_tensorflow_b200.utils import data_aug as D
    if not torch.cuda.is_available():
        raise SystemExit("augment_bench needs a GPU")
    card, power = _card()
    rng = np.random.default_rng(0)
    for n in a.batches:
        imgs = [rng.integers(0, 256, (375, 500, 3), dtype=np.uint8) for _ in range(n)]
        boxes = []
        for _ in range(n):
            xy = np.sort(rng.uniform(0, 370, (3, 2, 2)), axis=1)
            boxes.append(np.stack([xy[:, 0, 0], xy[:, 0, 1], xy[:, 1, 0] + 5, xy[:, 1, 1] + 5], 1).astype(np.float32))
        labels = [np.arange(3) for _ in range(n)]
        mix = _pairs(n, np.random.default_rng(1), random.Random(1))
        packed = D.PackedImages(imgs)
        np.random.seed(0); random.seed(0)
        params_seen = []
        orig = D._augment_launch

        def spy(pk, params):
            params_seen.append(params)
            return orig(pk, params)
        D._augment_launch = spy
        for _ in range(3):                                            # warm-up
            D.augment_train_batch(packed, boxes, labels, mix_with=mix)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.iters):
            D.augment_train_batch(packed, boxes, labels, mix_with=mix)
        torch.cuda.synchronize()
        dev_s = (time.perf_counter() - t0) / a.iters
        D._augment_launch = orig
        params = params_seen[-1]
        nbytes = _hbm_bytes(packed.desc, params)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 50
        D._augment_launch(packed, params)
        ev0.record()
        for _ in range(reps):
            D._augment_launch(packed, params)
        ev1.record()
        torch.cuda.synchronize()
        kern_s = ev0.elapsed_time(ev1) / 1e3 / reps
        host_s = None
        try:
            import cv2  # noqa: F401
            jobs = [(imgs[i], None if mix[i] is None else imgs[mix[i]],
                     np.concatenate([boxes[i], np.ones((3, 1), np.float32)], 1), 1000 + i) for i in range(n)]
            with Pool(os.cpu_count()) as pool:
                pool.map(_host_chain, jobs)                           # warm-up
                t0 = time.perf_counter()
                for _ in range(max(1, a.iters // 4)):
                    pool.map(_host_chain, jobs)
                host_s = (time.perf_counter() - t0) / max(1, a.iters // 4)
        except ImportError:
            pass
        print(json.dumps({
            "batch": n, "image": "375x500", "card": card, "power_limit": power, "host_cores": os.cpu_count(),
            "device_images_per_s": round(n / dev_s, 1), "device_batch_ms": round(dev_s * 1e3, 3),
            "launch_ms": round(kern_s * 1e3, 4), "hbm_bytes": nbytes,
            "launch_hbm_fraction": round(nbytes / HBM_BYTES_PER_S / kern_s, 3),
            "host_images_per_s": None if host_s is None else round(n / host_s, 1),
            "host_batch_ms": None if host_s is None else round(host_s * 1e3, 3)}))


if __name__ == "__main__":
    main()
