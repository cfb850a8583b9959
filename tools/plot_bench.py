"""Device drawing (plot_detections) against the host alternative at batch 64, from committed fixtures only.

  python tools/plot_bench.py [--batch 64] [--dets 20] [--iters 20]

Inputs: the VOC-size photographs of tools/jpeg_bench.py (375 x 500 and 500 x 375, tl 1), decoded on the device,
with --dets seeded labelled detections each.  Reports the card and its power limit, and:
- device: plot_detections(check=False) on the decoded batch, by CUDA events;
- host: D2H of the decoded batch, the reference's plot_one_box loop in cv2, H2D back (host clock, synchronised);
- chain: files -> decode_jpeg_batch -> preprocess_batch -> detect_raw -> restore_boxes -> plot_detections ->
  encode_jpeg_batch -> files, against the same chain drawing on the host (D2H, cv2, encode from the host images).
The host numbers need cv2; without it they are reported as not measured.  Exits nonzero if the device drawing differs
from cv2's."""
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
from tests import jpeg_cases, plot_cases  # noqa: E402
from yolov3_tensorflow_b200.utils.data_aug import (decode_jpeg_batch, encode_jpeg_batch, preprocess_batch,  # noqa: E402
                                                   restore_boxes)
from yolov3_tensorflow_b200.utils.plot_utils import get_color_table, plot_detections  # noqa: E402


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


def host_timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters


def cv2_plot_one_box(cv2, img, coord, label, color):
    """The reference's plot_one_box (utils/plot_utils.py), spelled out with cv2."""
    tl = int(round(0.002 * max(img.shape[0:2])))
    c1, c2 = (int(coord[0]), int(coord[1])), (int(coord[2]), int(coord[3]))
    cv2.rectangle(img, c1, c2, color, thickness=tl)
    tf = max(tl - 1, 1)
    t_size = cv2.getTextSize(label, 0, fontScale=float(tl) / 3, thickness=tf)[0]
    cv2.rectangle(img, c1, (c1[0] + t_size[0], c1[1] - t_size[1] - 3), color, -1)
    cv2.putText(img, label, (c1[0], c1[1] - 2), 0, float(tl) / 3, [0, 0, 0], thickness=tf, lineType=cv2.LINE_AA)


def cv2_draw(cv2, imgs, boxes, scores, labels, counts, table):
    for i, im in enumerate(imgs):
        for j in range(int(counts[i])):
            cv2_plot_one_box(cv2, im, boxes[i, j], plot_cases.COCO[labels[i, j]] +
                             ", {:.2f}%".format(scores[i, j] * 100), table[labels[i, j]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--dets", type=int, default=20)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "plot_bench needs a GPU"
    try:
        import cv2
    except ImportError:
        cv2 = None
    _, dec_cases = jpeg_cases.load()
    voc = [c["data"] for c in dec_cases if c["name"].startswith("voc_")]
    files = [voc[i % len(voc)] for i in range(a.batch)]
    packed = decode_jpeg_batch(files)
    n, k = a.batch, a.dets
    r = np.random.default_rng(0)
    boxes = np.zeros((n, k, 4), np.float32)
    for i, (_, h, w, _) in enumerate(packed.desc.tolist()):
        x, y = np.sort(r.uniform(0, w, (k, 2)), 1), np.sort(r.uniform(0, h, (k, 2)), 1)
        boxes[i] = np.stack([x[:, 0], y[:, 0], x[:, 1], y[:, 1]], 1)
    scores = r.random((n, k), dtype=np.float32)
    labels = r.integers(0, 80, (n, k)).astype(np.int32)
    counts = np.full(n, k, np.int32)
    table = get_color_table(80)
    dev = [torch.from_numpy(v).cuda() for v in (boxes, scores, labels, counts)]
    res = {"card": card(), "batch": n, "detections_per_image": k, "host_cores": os.cpu_count(),
           "images": "VOC-size q95 photographs (375 x 500, 500 x 375), tl 1"}
    ok = True

    clean = [packed.image(i).cpu().numpy() for i in range(n)]
    plot_detections(packed, *dev, plot_cases.COCO, table)
    if cv2 is not None:
        ref = [im.copy() for im in clean]
        cv2_draw(cv2, ref, boxes, scores, labels, counts, table)
        ok = all(np.array_equal(packed.image(i).cpu().numpy(), ref[i]) for i in range(n))
    t_dev = timed(lambda: plot_detections(packed, *dev, plot_cases.COCO, table, check=False), a.iters)
    res["device_draw_ms"] = t_dev * 1e3
    res["device_draw_img_s"] = n / t_dev

    # the host alternative for the same detections: D2H, the cv2 loop, H2D
    def host_draw():
        host = packed.data.cpu()
        imgs = [host[n * 32 + o: n * 32 + o + hh * p].numpy().reshape(hh, ww, 3).copy()
                for o, hh, ww, p in packed.desc.tolist()]
        cv2_draw(cv2, imgs, boxes, scores, labels, counts, table)
        return [torch.from_numpy(im).cuda(non_blocking=False) for im in imgs]
    if cv2 is not None:
        t_host = host_timed(host_draw, max(a.iters // 4, 2))
        res["host_draw_ms"] = t_host * 1e3
        res["host_draw_img_s"] = n / t_host
    else:
        res["host_draw"] = "not measured: cv2 does not import"

    from oracle import yolov3_oracle as O
    import yolov3_tensorflow_b200 as pkg
    m = pkg.yolov3(80, O.COCO_ANCHORS, dtype="fp16")
    m.set_params(O.make_params(80, seed=7, random_bn=True, det_scale=8.0, conf_bias=-2.0), "HWIO")

    def front():
        p = decode_jpeg_batch(files, check=False)
        x, params = preprocess_batch(p, 416, 416)
        _, ob, os_, ol, _, cnt = m.detect_raw(x, max_boxes=k, score_thresh=0.3, nms_thresh=0.45)
        cnt = cnt.clamp(max=k)
        # the seeded weights give some boxes far outside the image, past the int range cv2 accepts: keep both
        # chains on coordinates the reference can draw
        return p, restore_boxes(ob, cnt, params).clamp_(-1000.0, 5000.0), os_, ol, cnt

    def chain_device():
        p, b, s, lab, cnt = front()
        plot_detections(p, b, s, lab, cnt, plot_cases.COCO, table, check=False)
        return encode_jpeg_batch(p, quality=95)

    def chain_host():
        p, b, s, lab, cnt = front()
        imgs = [p.image(i).cpu().numpy() for i in range(n)]
        cv2_draw(cv2, imgs, b.cpu().numpy(), s.cpu().numpy(), lab.cpu().numpy(), cnt.cpu().numpy(), table)
        return encode_jpeg_batch(imgs, quality=95)
    res["chain_detections_per_image"] = float(front()[4].float().mean())
    t_chain = host_timed(chain_device, max(a.iters // 4, 2))
    res["chain_device_draw_img_s"] = n / t_chain
    if cv2 is not None:
        ok &= chain_device() == chain_host()
        t_chain_h = host_timed(chain_host, max(a.iters // 4, 2))
        res["chain_host_draw_img_s"] = n / t_chain_h
    else:
        res["chain_host_draw"] = "not measured: cv2 does not import"
    res["pixels_match_cv2"] = bool(ok) if cv2 is not None else "not checked: cv2 does not import"
    print(json.dumps(res))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
