"""Device k-means anchors (yolov3_tensorflow_b200.get_kmeans) against the vectorised numpy restatement on the host.

Workload: seeded COCO-like box sizes (w, h log-uniform in [4, 416]), k = 9, at --sizes rows (default 860,000, about
COCO train2017's box count, and 10,000,000).
  - device: get_kmeans from a numpy array (upload and input checks included) and from a CUDA tensor, host clock ending
    in the returned host values; best of --repeats.  Iteration count and time per iteration from the same clustering
    driven by KMeansSteps.run, less the initial draw on the host (timed apart); CUDA-event times of one assignment
    (with its [k + 1] read), one median and one avg_iou.
  - host: tests/kmeans_ref.py (whole-array numpy: the reference's arithmetic without its per-row Python loop).  At
    sizes up to --host-full rows it runs to convergence and the anchors and average IoU must be equal; above that it
    runs --host-iters iterations and the clusters must equal the device's after the same number of updates.

    python tools/kmeans_bench.py [--sizes 860000 10000000] [--repeats 3] [--host-full 1000000] [--host-iters 2]
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

from tests import kmeans_ref as K  # noqa: E402
from yolov3_tensorflow_b200 import get_kmeans as G  # noqa: E402

KC, SEED = 9, 1234


def _card():
    try:
        return subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", "--query-gpu=name,power.limit",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return f"{torch.cuda.get_device_name()}, unknown"


def _best(fn, repeats):
    best, val = float("inf"), None
    for _ in range(repeats):
        torch.cuda.synchronize()
        t = time.perf_counter()
        val = fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t)
    return best, val


def _event_ms(fn, reps=20):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def bench_size(rows, args):
    boxes = K.gen_float_boxes(SEED + rows, rows)
    dev = torch.from_numpy(boxes).cuda()
    r = {"rows": rows, "k": KC}
    t_np, (anchors, ave) = _best(lambda: G.get_kmeans(boxes, KC, seed=SEED), args.repeats)
    t_dev, (anchors_d, ave_d) = _best(lambda: G.get_kmeans(dev, KC, seed=SEED), args.repeats)
    assert (anchors_d, ave_d) == (anchors, ave)
    s = G.KMeansSteps(dev, KC)
    t_run, iters = _best(lambda: s.run(SEED), 1)
    # the reference's draw, choice(rows, k, replace=False), permutes all rows on the host: timed apart
    t_draw, _ = _best(lambda: np.random.RandomState(SEED).choice(rows, KC, replace=False), 1)
    r.update(device_get_kmeans_s_from_numpy=round(t_np, 4), device_get_kmeans_s_from_cuda=round(t_dev, 4),
             iterations=iters, device_loop_s=round(t_run, 4), host_draw_s=round(t_draw, 4),
             device_ms_per_iteration=round(1e3 * (t_run - t_draw) / iters, 4),
             assign_and_read_ms=round(_event_ms(s.assign), 4), median_ms=round(_event_ms(s.median), 4),
             avg_iou_ms=round(_event_ms(s.avg_iou), 4), anchors=anchors, avg_iou=float(ave))
    init = K.initial_clusters(boxes, KC, SEED)
    if rows <= args.host_full:
        t = time.perf_counter()
        h_anchors, h_ave = K.get_kmeans(boxes, KC, SEED)
        t_host = time.perf_counter() - t                                  # the draw included
        r.update(host_get_kmeans_s=round(t_host, 2), host_ms_per_iteration=round(1e3 * t_host / iters, 1),
                 anchors_equal=h_anchors == anchors, avg_iou_equal=bool(h_ave == ave))
    else:
        t = time.perf_counter()
        c = init
        for it in range(args.host_iters):
            c = K.medians(boxes, K.assign(boxes, c), KC, it + 1)
        t_host = time.perf_counter() - t
        s.set_clusters(init)
        for _ in range(args.host_iters):
            s.assign()
            s.median()
        got = s.clusters.cpu().numpy()
        r.update(host_iterations_run=args.host_iters, host_ms_per_iteration=round(1e3 * t_host / args.host_iters, 1),
                 clusters_equal_after_host_iterations=bool(np.array_equal(got.view(np.uint64), c.view(np.uint64))))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[860_000, 10_000_000])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--host-full", type=int, default=1_000_000)
    ap.add_argument("--host-iters", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "kmeans_bench needs a GPU"
    G.get_kmeans(K.gen_float_boxes(0, 5000), KC, seed=0)          # module load and first launches
    out = {"card": _card(), "results": [bench_size(n, args) for n in args.sizes]}
    ok = all(r.get("anchors_equal", True) and r.get("avg_iou_equal", True) and
             r.get("clusters_equal_after_host_iterations", True) for r in out["results"])
    out["agree"] = ok
    print(json.dumps(out))
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
