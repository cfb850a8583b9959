"""The fused detection step against the three-call pipeline at custom class counts, on one GPU.

Workload: batch 64, 416 x 416, cfg-2 weights (bench.make_bench_params over the model's own conv table: Glorot-uniform,
identity BN, heads x 8, conf bias -2), max_boxes 200, score 0.3, NMS 0.45, fp16, for C in --classes.  Per class count
the two paths alternate, `--runs` runs each, on the same device-resident batch:
  - fused : model.detect_raw (decode and score filter inside the detection-head epilogues, one engine call);
  - three : forward() -> predict_scores() -> batched_nms_raw() (float32 head maps and an [n, B, C] score tensor in HBM).
Each run: `--warmup` untimed steps, then CUDA events around `--steps` steps; ms per step.  The two paths' detections are
checked to be the same bits before timing; the tool exits with an error if they are not.  `detections` is the number
kept by the NMS over the batch: 0 means no score reached the threshold, so that row times an NMS with no work.

    python tools/detect_classes_bench.py [--classes 1,3,20,43,80] [--steps 20] [--warmup 3] [--runs 3] [--batch 64]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--classes", default="1,3,20,43,80")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--size", type=int, default=416)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("detect_classes_bench needs a CUDA device")
    import bench
    import yolov3_tensorflow_b200 as pkg
    from tests.synth import gen_inputs
    from yolov3_tensorflow_b200 import _lib
    from yolov3_tensorflow_b200.utils.nms_utils import batched_nms_raw

    B, S = args.batch, args.size
    anchors = pkg.parse_anchors(os.path.join(ROOT, "yolov3_tensorflow_b200", "data", "yolo_anchors.txt"))
    x = torch.from_numpy(gen_inputs(0, B, S, S)).cuda()
    rows = []
    for cn in (int(c) for c in args.classes.split(",")):
        m = pkg.yolov3(cn, anchors, dtype="fp16")
        m.set_params(bench.make_bench_params(specs=m.conv_table(cn)), "HWIO")

        def three():
            boxes, scores = m.predict_scores(m.forward(x))
            return (boxes,) + tuple(batched_nms_raw(boxes, scores, cn, NMS["max_boxes"], NMS["score_thresh"],
                                                    NMS["nms_thresh"]))

        def fused():
            return m.detect_raw(x, **NMS)

        f, t = fused(), three()
        supported = int(_lib.lib.yb_net_detect_supported(m._last_plan.handle))
        counts = t[5].tolist()
        same = torch.equal(f[0], t[0]) and torch.equal(f[5], t[5]) and all(
            torch.equal(a[i, :k], b[i, :k]) for a, b in zip(f[1:5], t[1:5]) for i, k in enumerate(counts))
        if not same:
            raise SystemExit(f"detect_classes_bench: {cn} classes: the fused and the three-call detections differ")
        runs = {"fused": [], "three": []}
        for _ in range(args.runs):
            runs["fused"].append(_time(fused, args.steps, args.warmup))
            runs["three"].append(_time(three, args.steps, args.warmup))
        fm, tm = float(np.mean(runs["fused"])), float(np.mean(runs["three"]))
        rows.append({"classes": cn, "fused_supported": supported, "same_bits": True, "detections": sum(counts),
                     "nms_has_work": sum(counts) > 0,
                     "fused_ms": runs["fused"], "three_ms": runs["three"], "fused_ms_mean": fm, "three_ms_mean": tm,
                     "three_over_fused": tm / fm})
        del m
        torch.cuda.empty_cache()
    out = {"workload": f"detect_raw vs forward+predict_scores+batched_nms_raw, batch {B} {S}x{S} fp16 cfg-2 weights",
           "card": _card(), "steps": args.steps, "warmup": args.warmup, "rows": rows}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
