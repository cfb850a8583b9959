"""The training resize (utils.data_aug.resize_train_batch: host tap tables, one table copy, one
yb_resize_batch_interp launch) on training-like crops: augment_train_batch's output for 375 x 500 images, letterboxed
to 416 x 416 and 608 x 608 at batch 32 and 64.  For each interpolation alone (0..4) and for the batch's own drawn mix,
prints one JSON line with the launch time (CUDA events over many launches after warm-up; the host table build and
its H2D copy are reported apart), its share of the HBM bound (crop bytes read + float32 output written + tables, over
3.35 TB/s), and the host reference: cv2.resize + cvtColor(BGR2RGB) + float32 / 255 of the same crops, timed on one
core and divided by the host's core count for an ideal all-core figure.  The card's name and power limit are read
in the same run.
Usage: python tools/resize_interp_bench.py [--batches 32 64] [--sizes 416 608] [--iters 50]"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

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


def _host_one(args):
    """letterbox_resize(img, S, S, interp) + cvtColor(BGR2RGB) + float32 / 255 with cv2 (default build, IPP on)."""
    import cv2
    img, s, interp = args
    h, w = img.shape[:2]
    ratio = min(s / w, s / h)
    rw, rh = int(ratio * w), int(ratio * h)
    padded = np.full((s, s, 3), 128, np.uint8)
    dw, dh = int((s - rw) / 2), int((s - rh) / 2)
    padded[dh: dh + rh, dw: dw + rw] = cv2.resize(img, (rw, rh), interpolation=interp)
    return (cv2.cvtColor(padded, cv2.COLOR_BGR2RGB).astype(np.float32) / 255.).nbytes


def _crops(n):
    """augment_train_batch's crops of n 375 x 500 images (half mixed up) -> (PackedImages, interp)."""
    from yolov3_tensorflow_b200.utils import data_aug as D
    rng = np.random.default_rng(0)
    imgs = [rng.integers(0, 256, (375, 500, 3), dtype=np.uint8) for _ in range(n)]
    boxes = [np.array([[50, 60, 300, 330], [200, 10, 480, 200]], np.float32) for _ in range(n)]
    labels = [np.arange(2) for _ in range(n)]
    mix = [(i + 1) % n if i % 2 == 0 else None for i in range(n)]
    np.random.seed(0)
    random.seed(0)
    packed, _, _, interp, _ = D.augment_train_batch(imgs, boxes, labels, mix_with=mix)
    keep = [i for i in range(n) if packed.desc[i, 1] > 0 and packed.desc[i, 2] > 0]
    assert len(keep) == n, "an empty crop in the benchmark batch"
    return packed, interp


def _time(fn, iters):
    import torch
    for _ in range(5):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--sizes", type=int, nargs="+", default=[416, 608])
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    import ctypes as C

    import torch
    from yolov3_tensorflow_b200._lib import check, lib, ptr, stream_handle
    from yolov3_tensorflow_b200.utils import data_aug as D
    if not torch.cuda.is_available():
        raise SystemExit("resize_interp_bench needs a GPU")
    card, power = _card()
    procs = os.cpu_count() or 1
    import cv2
    cv2.setNumThreads(1)                               # the host reference is timed on one core
    for n in a.batches:
        packed, drawn = _crops(n)
        host_imgs = [packed.image(i).cpu().numpy() for i in range(n)]
        src_bytes = int(sum(3 * h * w for h, w in packed.desc[:, 1:3].tolist()))
        desc = np.ascontiguousarray(packed.desc)
        for s in a.sizes:
            out = torch.empty((n, s, s, 3), dtype=torch.float32, device="cuda")
            params = torch.empty((n, 4), dtype=torch.float64, device="cuda")
            for name, interp in [(str(k), np.full(n, k, np.int32)) for k in range(5)] + [("mixed", drawn)]:
                it = np.ascontiguousarray(interp, np.int32)
                dp, ip = desc.ctypes.data_as(C.c_void_p), it.ctypes.data_as(C.c_void_p)
                nb = C.c_size_t()
                t0 = time.perf_counter()
                check(lib.yb_resize_tables_bytes(dp, n, s, s, 1, ip, C.byref(nb)))
                host = torch.empty((nb.value,), dtype=torch.uint8, pin_memory=True)
                check(lib.yb_resize_tables(dp, n, s, s, 1, ip, C.c_void_p(host.data_ptr()), nb.value))
                table_ms = (time.perf_counter() - t0) * 1e3
                tabs = host.to("cuda", non_blocking=True)

                def launch():
                    check(lib.yb_resize_batch_interp(ptr(packed.pixels), packed.pixels.numel(), dp,
                                                     ptr(packed.desc_dev), n, s, s, 1, ip,
                                                     C.c_void_p(host.data_ptr()), ptr(tabs), nb.value, ptr(out),
                                                     ptr(params), stream_handle()), "yb_resize_batch_interp")
                ms = _time(launch, a.iters)
                full_ms = _time(lambda: D.resize_train_batch(packed, s, s, interp, out=out), a.iters)
                moved = src_bytes + out.numel() * 4 + nb.value
                jobs = [(img, s, int(k)) for img, k in zip(host_imgs, interp.tolist())]
                for job in jobs[:4]:
                    _host_one(job)
                t0 = time.perf_counter()
                for job in jobs:
                    _host_one(job)
                host_ms = (time.perf_counter() - t0) * 1e3
                print(json.dumps({"batch": n, "size": s, "interp": name, "launch_ms": round(ms, 4),
                                  "hbm_bound_share": round(moved / HBM_BYTES_PER_S * 1e3 / ms, 3),
                                  "bytes_moved": moved, "table_bytes": nb.value,
                                  "table_build_ms": round(table_ms, 3),
                                  "resize_train_batch_ms": round(full_ms, 4),
                                  "host_cv2_ms_one_core": round(host_ms, 3),
                                  "host_cv2_ms_all_cores_ideal": round(host_ms / procs, 3), "host_cores": procs,
                                  "card": card, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
