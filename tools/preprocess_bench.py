"""The evaluation input path, uint8 on the device (utils.data_aug.preprocess_batch) against the host path (cv2 resize +
BGR->RGB + float32 / 255 per image, float32 upload), both feeding detect_raw.

Workload: --batch seeded uint8 BGR sources of VOC's two common shapes (500 x 375 and 375 x 500, alternating), resized to
--size x --size with the reference's evaluation interpolation (INTER_LINEAR), stretched (eval.py / eval_voc.py's
default) and letterboxed; cfg-2 weights, fp16, detect_raw at the evaluation settings (400 per class, score 0.01,
NMS 0.45).
  - A: preprocess_batch (pack into one pinned buffer, one H2D copy, one launch) -> detect_raw
  - B: cv2.resize + cvtColor + np.float32 / 255 per image on the host, np.stack, one float32 upload -> detect_raw
    (the numpy restatement of tests/resize_ref.py when cv2 is missing; the JSON says which)
Per batch: host clock around the whole path ending in a synchronise, median and minimum over --batches after --warmup.
The resize kernel alone: CUDA events over --kernel-reps launches on the uploaded batch.  Bytes over PCIe are the
host -> device copies each path makes.  The inputs and the detections (every valid slot of boxes, scores, labels and
the counts) of the two paths are compared byte for byte.

    python tools/preprocess_bench.py [--batch 64] [--size 416] [--batches 20] [--warmup 3]
Prints one JSON line, with the card name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        return subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", "--query-gpu=name,power.limit",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return f"{torch.cuda.get_device_name()}, unknown"


def _sources(n, seed=17):
    """Smooth-ish uint8 BGR images: a coarse random field upsampled, plus noise (compresses like a photo would not
    matter here; what matters is that the bench weights produce detections)."""
    rng = np.random.default_rng(seed)
    imgs = []
    for i in range(n):
        h, w = (375, 500) if i % 2 == 0 else (500, 375)
        coarse = rng.integers(0, 256, (h // 25 + 2, w // 25 + 2, 3)).astype(np.float32)
        img = np.repeat(np.repeat(coarse, 25, 0), 25, 1)[:h, :w]
        img = np.clip(img + rng.normal(0, 12, img.shape), 0, 255).astype(np.uint8)
        imgs.append(np.ascontiguousarray(img))
    return imgs


def _host_input(imgs, size, letterbox, cv2):
    from tests import resize_ref as R
    xs = []
    for img in imgs:
        if cv2 is None:
            xs.append(R.preprocess(img, size, size, letterbox, 1)[0])
            continue
        if letterbox:                                   # utils/data_aug.letterbox_resize(interp=1)
            h, w = img.shape[:2]
            ratio = min(size / w, size / h)
            rw, rh = int(ratio * w), int(ratio * h)
            pad = np.full((size, size, 3), 128, np.uint8)
            dw, dh = int((size - rw) / 2), int((size - rh) / 2)
            pad[dh: rh + dh, dw: rw + dw] = cv2.resize(img, (rw, rh), interpolation=1)
        else:
            pad = cv2.resize(img, (size, size), interpolation=1)
        xs.append(np.asarray(cv2.cvtColor(pad, cv2.COLOR_BGR2RGB), np.float32) / 255.)
    return np.stack(xs).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--size", type=int, default=416)
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kernel-reps", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("preprocess_bench needs a GPU")
    try:
        import cv2
    except ImportError:
        cv2 = None
    import bench
    import yolov3_tensorflow_b200 as pkg
    from oracle import yolov3_oracle as O
    from yolov3_tensorflow_b200.utils import data_aug as A

    torch.cuda.set_device(0)
    m = pkg.yolov3(80, O.COCO_ANCHORS, dtype="fp16")
    m.set_params(bench.make_bench_params(specs=m.conv_table(80)), "HWIO")
    imgs = _sources(args.batch)
    S = args.size
    det_kw = dict(max_boxes=400, score_thresh=0.01, nms_thresh=0.45)
    line = {"card": _card(), "batch": args.batch, "size": S, "sources": "500x375 / 375x500 uint8 BGR",
            "host_resize": "cv2 " + cv2.__version__ if cv2 is not None else "numpy restatement"}

    def path_a(letterbox):
        x, _ = A.preprocess_batch(imgs, S, S, letterbox=letterbox, interp=1)
        return x, m.detect_raw(x, **det_kw)

    def path_b(letterbox):
        x = torch.from_numpy(_host_input(imgs, S, letterbox, cv2)).cuda()
        return x, m.detect_raw(x, **det_kw)

    for letterbox in (False, True):
        mode = "letterbox" if letterbox else "stretch"
        res = {}
        outs = {}
        for name, fn in (("A_device_uint8", path_a), ("B_host_cv2_float32", path_b)):
            for _ in range(args.warmup):
                fn(letterbox)
            torch.cuda.synchronize()
            ts = []
            for _ in range(args.batches):
                t0 = time.perf_counter()
                x, out = fn(letterbox)
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t0)
            outs[name] = (x.cpu().numpy(), [t.cpu().numpy() for t in out[1:]])
            res[name] = {"ms_per_batch_median": round(1e3 * float(np.median(ts)), 3),
                         "ms_per_batch_min": round(1e3 * min(ts), 3)}
        packed = A.PackedImages(imgs)
        res["A_device_uint8"]["h2d_bytes"] = packed.h2d_bytes
        res["B_host_cv2_float32"]["h2d_bytes"] = int(args.batch * S * S * 3 * 4)
        # detect_raw alone on the same input, for the share the input path takes
        xa = torch.from_numpy(outs["A_device_uint8"][0]).cuda()
        for _ in range(args.warmup):
            m.detect_raw(xa, **det_kw)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.batches):
            m.detect_raw(xa, **det_kw)
        e1.record()
        e1.synchronize()
        res["detect_raw_only_ms"] = round(e0.elapsed_time(e1) / args.batches, 3)
        # the resize kernel alone (packed batch already on the device)
        out = torch.empty((args.batch, S, S, 3), dtype=torch.float32, device="cuda")
        for _ in range(10):
            A._resize_packed(packed, S, S, letterbox, 1, out)
        e0.record()
        for _ in range(args.kernel_reps):
            A._resize_packed(packed, S, S, letterbox, 1, out)
        e1.record()
        e1.synchronize()
        k_us = 1e3 * e0.elapsed_time(e1) / args.kernel_reps
        moved = packed.pixels.numel() + out.numel() * 4        # every source byte read once, every output written once
        res["resize_kernel_us"] = round(k_us, 2)
        res["resize_kernel_gb_per_s"] = round(moved / (k_us * 1e-6) / 1e9, 1)
        xa_np, oa = outs["A_device_uint8"]
        xb_np, ob = outs["B_host_cv2_float32"]
        same = xa_np.tobytes() == xb_np.tobytes() and oa[4].tobytes() == ob[4].tobytes()
        for i, k in enumerate(oa[4].tolist()):
            for ta, tb in zip(oa[:3], ob[:3]):
                same = same and ta[i, :k].tobytes() == tb[i, :k].tobytes()
        res["inputs_and_detections_byte_identical"] = bool(same)
        res["detections"] = int(oa[4].sum())
        line[mode] = res
    print(json.dumps(line))


if __name__ == "__main__":
    main()
