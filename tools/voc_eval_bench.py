"""Device VOC evaluation (utils.eval_utils.VOCEvaluator) against the host path (get_preds_gpu rows + voc_eval per class).

Workload: seeded synthetic validation sets in the [n, cap] NMS layout, 80 classes, 7 ground-truth boxes per image;
half of the detections are jittered copies of a ground-truth box (mostly of its class), the rest are random boxes.
  - device: every add_batch (64 images each) plus result(), host clock ending in a synchronise, at --images images
    x 300 and x 2000 detections per image, and at the host set's size; best of --repeats.
  - host: on --host-images x 2000 detections (scores distinct, so voc_eval's unstable sort cannot reorder ties): the
    rows get_preds_gpu builds (copy to the host + one Python list per detection), then voc_eval for each class.
    Both paths must give the same results (area AP within 1e-12, everything else exact).
  - context: detect_raw at the reference's evaluation settings (400 per class, score 0.01, NMS 0.45; cfg-2 weights,
    batch 64, 416 x 416) for --images images, CUDA events.

    python tools/voc_eval_bench.py [--images 5000] [--host-images 1000] [--repeats 3]
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

C = 80
BATCH = 64


def _card():
    try:
        return subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", "--query-gpu=name,power.limit",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return f"{torch.cuda.get_device_name()}, unknown"


def _synthetic_set(seed, n, k, distinct_scores=False):
    """Device tensors (out_boxes [n,k,4], out_scores, out_labels [n,k], counts [n]) in NMS order, gt on the host."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"
    gxy = torch.rand((n, 7, 2), generator=g, device=dev, dtype=torch.float64) * 380
    gwh = 8 + torch.rand((n, 7, 2), generator=g, device=dev, dtype=torch.float64) * 120
    gt_boxes = torch.cat([gxy, gxy + gwh], 2)
    gt_labels = torch.randint(0, C, (n, 7), generator=g, device=dev, dtype=torch.int32)
    src = torch.randint(0, 7, (n, k), generator=g, device=dev)
    near = torch.rand((n, k), generator=g, device=dev) < 0.5
    jit = (torch.rand((n, k, 4), generator=g, device=dev, dtype=torch.float64) - 0.5) * 0.6
    gsrc = torch.gather(gt_boxes, 1, src[..., None].expand(n, k, 4))
    wh = (gsrc[..., 2:] - gsrc[..., :2]).repeat(1, 1, 2)
    rnd_xy = torch.rand((n, k, 2), generator=g, device=dev, dtype=torch.float64) * 380
    rnd = torch.cat([rnd_xy, rnd_xy + 8 + torch.rand((n, k, 2), generator=g, device=dev, dtype=torch.float64) * 120], 2)
    boxes = torch.where(near[..., None], gsrc + jit * wh, rnd).float()
    labels = torch.randint(0, C, (n, k), generator=g, device=dev, dtype=torch.int32)
    keep = near & (torch.rand((n, k), generator=g, device=dev) < 0.85)
    labels = torch.where(keep, torch.gather(gt_labels, 1, src), labels)
    if distinct_scores:            # distinct multiples of 2^-23: exact in float32, no ties anywhere in the set
        scores = ((torch.randperm(1 << 23, generator=g, device=dev)[:n * k] + 1).double() * 2.0 ** -23).reshape(n, k)
    else:
        scores = torch.randint(1, 1 << 23, (n, k), generator=g, device=dev).double() * 2.0 ** -23
    order = torch.argsort(labels.double() * 2 - scores, dim=1, stable=True)       # class ascending, score descending
    boxes = torch.gather(boxes, 1, order[..., None].expand(n, k, 4)).contiguous()
    scores = torch.gather(scores.float(), 1, order).contiguous()
    labels = torch.gather(labels, 1, order).contiguous()
    counts = torch.full((n,), k, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    return (boxes, scores, labels, counts), (gt_boxes.cpu(), gt_labels.cpu(), torch.full((n,), 7, dtype=torch.int32))


def _device_eval(dets, gts, repeats):
    from yolov3_tensorflow_b200.utils.eval_utils import VOCEvaluator
    n = dets[0].shape[0]
    gb, gl, gc = (t.pin_memory() for t in gts)
    ev = VOCEvaluator(C)
    best, res = float("inf"), None
    for _ in range(repeats + 1):                 # the first pass warms up (module load, pool growth)
        ev.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for s in range(0, n, BATCH):
            ev.add_batch(*(t[s:s + BATCH] for t in dets), gb[s:s + BATCH], gl[s:s + BATCH], gc[s:s + BATCH])
        res = ev.result(False)
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best, res, len(ev)


def _host_eval(dets, gts):
    from yolov3_tensorflow_b200.utils.eval_utils import voc_eval
    n = dets[0].shape[0]
    t0 = time.perf_counter()
    rows = []
    for s in range(0, n, BATCH):                 # get_preds_gpu: copy one batch's kept detections, one list per row
        ks = dets[3][s:s + BATCH].cpu().tolist()
        ob, os_, ol = (t[s:s + BATCH].cpu().numpy() for t in dets[:3])
        for i, k in enumerate(ks):
            b, sc, lb = ob[i, :k], os_[i, :k], ol[i, :k]
            for j in range(k):
                rows.append([s + i, b[j, 0], b[j, 1], b[j, 2], b[j, 3], sc[j], lb[j]])
    t1 = time.perf_counter()
    gb, gl, gc = (t.numpy() for t in gts)
    gt_dict = {i: [[float(v) for v in gb[i, j]] + [int(gl[i, j])] for j in range(int(gc[i]))] for i in range(n)}
    with np.errstate(divide="ignore", invalid="ignore"):
        res = [voc_eval(gt_dict, rows, c, 0.5, False) for c in range(C)]
    t2 = time.perf_counter()
    return t1 - t0, t2 - t1, res


def _same(a, b):
    for x, y in zip(a, b):
        x, y = np.asarray([float(v) for v in x]), np.asarray([float(v) for v in y])
        if not (np.array_equal(x[:4], y[:4], equal_nan=True) and (np.isnan(x[4]) == np.isnan(y[4]))
                and (np.isnan(x[4]) or abs(x[4] - y[4]) <= 1e-12)):
            return False
    return len(a) == len(b)


def _detect_raw_s(images):
    import bench
    import yolov3_tensorflow_b200 as pkg
    from tests.synth import gen_inputs
    anchors = pkg.parse_anchors(os.path.join(ROOT, "yolov3_tensorflow_b200", "data", "yolo_anchors.txt"))
    m = pkg.yolov3(C, anchors, dtype="fp16")
    m.set_params(bench.make_bench_params(specs=m.conv_table(C)), "HWIO")
    x = torch.from_numpy(gen_inputs(0, BATCH, 416, 416)).cuda()
    nms = dict(max_boxes=400, score_thresh=0.01, nms_thresh=0.45)
    out = m.detect_raw(x, **nms)
    steps = -(-images // BATCH)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        out = m.detect_raw(x, **nms, out=out)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 * images / (steps * BATCH), int(out[5].sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--host-images", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("voc_eval_bench needs a CUDA device")
    out = {"workload": f"{C} classes, 7 gt per image, add_batch per {BATCH} images + result()", "card": _card()}
    dev = {}
    for k in (300, 2000):
        dets, gts = _synthetic_set(k, args.images, k)
        s, _, nd = _device_eval(dets, gts, args.repeats)
        dev[f"{args.images}x{k}"] = {"detections": nd, "device_s": s, "device_ms_per_million": s * 1e3 / (nd / 1e6)}
        del dets
    dets, gts = _synthetic_set(7, args.host_images, 2000, distinct_scores=True)
    s, dres, nd = _device_eval(dets, gts, args.repeats)
    rows_s, voc_s, hres = _host_eval(dets, gts)
    out["device"] = dev
    out["host_set"] = {"detections": nd, "device_s": s, "host_rows_s": rows_s, "host_voc_eval_s": voc_s,
                       "host_total_s": rows_s + voc_s, "speedup": (rows_s + voc_s) / s, "results_equal": _same(dres, hres),
                       "mAP": float(np.mean([r[4] for r in dres]))}
    det_s, kept = _detect_raw_s(args.images)
    out["detect_raw"] = {"images": args.images, "seconds": det_s, "detections_last_batch": kept}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
