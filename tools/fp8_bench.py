"""Calibrated fp8 (e4m3) inference against fp16 on one GPU: speed and agreement.

Workload: bench.py's flagship step (80 classes, batch 64, 416 x 416, cfg-2 weights from bench.make_bench_params,
detect_raw with max_boxes 200, score 0.3, NMS 0.45).  The fp16 model is quantized with quantize_fp8() on one seeded
calibration batch (gen_inputs seed 1000), different from the timed batch (seed 0).  The two models alternate, 3 runs
each, in one process; every run measures
  - step_ms : detect_raw on the device-resident batch, CUDA events around `--steps` steps;
  - conv_ms : the 74 tensor-core convs alone (detect_raw phases=2), events around each, mean over `--steps` steps;
  - graphed_ms : single-image detect_graphed latency (CUDA-graph replay), events around each, mean over `--steps` calls.
Agreement: the fp8 detections of the timed batch scored against the fp16 detections of the same images as ground truth
(utils.eval_utils.voc_eval, IoU 0.5), mean AP over the classes the fp16 model detects.  With random weights this
measures how much the quantization moves the detections, not accuracy on real data.

    python tools/fp8_bench.py [--steps 20] [--warmup 3] [--runs 3] [--batch 64] [--size 416]
Prints one JSON line, with the card name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NMS = dict(max_boxes=200, score_thresh=0.3, nms_thresh=0.45)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", "--query-gpu=name,power.limit",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = f"{torch.cuda.get_device_name()}, unknown"
    return out


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def _conv_ms(model, x, steps, warmup):
    res = model.detect_raw(x, **NMS)
    ms = []
    for i in range(steps + warmup):
        b, c = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        model.detect_raw(x, **NMS, phases=1, out=res)
        b.record()
        model.detect_raw(x, **NMS, phases=2, out=res)
        c.record()
        model.detect_raw(x, **NMS, phases=4, out=res)
        torch.cuda.synchronize()
        if i >= warmup:
            ms.append(b.elapsed_time(c))
    return float(np.mean(ms))


def _detections(model, x):
    """[(img, x0, y0, x1, y1, score, label)] rows of every image (get_preds_gpu's format)."""
    _, ob, os_, ol, _, cnt = model.detect_raw(x, **NMS)
    ob, os_, ol, cnt = ob.cpu().numpy(), os_.cpu().numpy(), ol.cpu().numpy(), cnt.cpu().numpy()
    rows = []
    for i, k in enumerate(cnt):
        for j in range(int(k)):
            rows.append([i] + [float(v) for v in ob[i, j]] + [float(os_[i, j]), int(ol[i, j])])
    return rows


def _agreement(ref_rows, rows, num_images):
    from yolov3_tensorflow_b200.utils.eval_utils import voc_eval
    gt = {i: [] for i in range(num_images)}
    for r in ref_rows:
        gt[r[0]].append(r[1:5] + [r[6]])
    classes = sorted({r[6] for r in ref_rows})
    aps = [voc_eval(gt, rows, c, 0.5)[4] for c in classes]
    return float(np.mean(aps)) if aps else float("nan"), len(classes)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--size", type=int, default=416)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_bench needs a CUDA device")
    import bench
    import yolov3_tensorflow_b200 as pkg
    from tests.synth import gen_inputs

    B, S = args.batch, args.size
    anchors = pkg.parse_anchors(os.path.join(ROOT, "yolov3_tensorflow_b200", "data", "yolo_anchors.txt"))
    m16 = pkg.yolov3(80, anchors, dtype="fp16")
    m16.set_params(bench.make_bench_params(specs=m16.conv_table(80)), "HWIO")
    x = torch.from_numpy(gen_inputs(0, B, S, S)).cuda()
    calib = torch.from_numpy(gen_inputs(1000, B, S, S)).cuda()
    m8 = m16.quantize_fp8(calib)
    x1 = x[:1].clone()
    runs = {"fp16": [], "fp8": []}
    for _ in range(args.runs):
        for name, m in (("fp16", m16), ("fp8", m8)):
            step = _time(lambda: m.detect_raw(x, **NMS), args.steps, args.warmup)
            conv = _conv_ms(m, x, args.steps, args.warmup)
            graphed = _time(lambda: m.detect_graphed(x1, **NMS), args.steps, args.warmup)
            runs[name].append({"step_ms": step, "img_per_s": B / step * 1e3, "conv_ms": conv, "graphed_ms": graphed})
    ref_rows, rows = _detections(m16, x), _detections(m8, x)
    mAP, ncls = _agreement(ref_rows, rows, B)
    out = {"workload": f"detect_raw batch {B} {S}x{S} cfg-2 weights, 80 classes", "card": _card(),
           "steps": args.steps, "warmup": args.warmup, "runs": runs,
           "conv_ms_fp16_mean": float(np.mean([r["conv_ms"] for r in runs["fp16"]])),
           "conv_ms_fp8_mean": float(np.mean([r["conv_ms"] for r in runs["fp8"]])),
           "agreement_map_vs_fp16": mAP, "agreement_classes": ncls,
           "detections_fp16": len(ref_rows), "detections_fp8": len(rows)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
