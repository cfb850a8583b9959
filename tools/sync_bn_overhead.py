"""Host and launch cost of the layered (synchronised-BN) training step on one GPU.

Times the fused train_step against train_step_sync_bn driven with an identity exchange (bn_replicas = 1, nothing
all-reduced), alternating the two step by step on one model, with CUDA events around every step.  Both compute the
same step; the difference is what the per-layer calls, the 2 x 72 exchange points and the Python generator cost.
The multi-GPU exchange itself (the all-reduces) is not part of this measurement.

    python tools/sync_bn_overhead.py [--size 416] [--batch 32] [--dtype bf16] [--steps 50] [--warmup 5]
Prints one JSON line with the card name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", "--query-gpu=power.limit",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def _identity(gen):
    reply = None
    try:
        while True:
            kind, _ = gen.send(reply)
            reply = 1.0 if kind == "grad_scale" else None
    except StopIteration as done:
        return done.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=416)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--dtype", default="bf16")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sync_bn_overhead: needs a CUDA device")
    import yolov3_tensorflow_b200 as pkg
    from oracle import yolov3_oracle as O
    m = pkg.yolov3(80, O.COCO_ANCHORS, dtype=a.dtype)
    m.init_params(seed=0)
    n, s = a.batch, a.size
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand((n, s, s, 3), generator=g, device="cuda")
    ys = [torch.zeros((n, s // d, s // d, 3, 86), device="cuda") for d in (32, 16, 8)]
    lr = 1e-5

    def fused():
        m.train_step(x, ys, lr)

    def layered():
        _identity(m.train_step_sync_bn(x, ys, lr, bn_replicas=1))

    runs = {"fused": fused, "layered": layered}
    for _ in range(a.warmup):
        for f in runs.values():
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    for _ in range(a.steps):
        for k, f in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1))
    name, power = _card()
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(json.dumps({
        "card": name, "power_limit": power, "size": s, "batch": n, "dtype": a.dtype, "steps": a.steps,
        "fused_ms_median": round(med["fused"], 3), "layered_ms_median": round(med["layered"], 3),
        "fused_ms_p10_p90": [round(float(np.percentile(times["fused"], q)), 3) for q in (10, 90)],
        "layered_ms_p10_p90": [round(float(np.percentile(times["layered"], q)), 3) for q in (10, 90)],
        "overhead_ms": round(med["layered"] - med["fused"], 3),
        "overhead_pct": round(100 * (med["layered"] / med["fused"] - 1), 2)}))


if __name__ == "__main__":
    main()
