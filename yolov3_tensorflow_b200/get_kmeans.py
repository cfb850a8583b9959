"""k-means anchors for YOLOv3 (the reference's get_kmeans.py), with the clustering on the GPU.

`kmeans` and `avg_iou` return what the reference's functions return, bit for bit: the same float64 IoU, the same
`np.argmin` assignment, the same per-cluster `np.median` and the same pairwise sum in the mean.  Each Lloyd iteration is
one assignment launch (yb_kmeans_assign), one [k + 1] int32 read on the host (counts and changes), then one median
launch (yb_kmeans_median, a radix select, so no sort).  The initial clusters are drawn on the host, as the reference
draws them: `np.random.RandomState(seed).choice(rows, k, replace=False)`.

One divergence: when a cluster becomes empty the reference's loop never returns (np.median of nothing is NaN and every
box then moves to the NaN cluster); here `kmeans` raises ValueError naming the cluster and the iteration.

    python -m yolov3_tensorflow_b200.get_kmeans train.txt [--target-size W H | --original-size] [--clusters 9]
                                                          [--seed S]
"""
from __future__ import annotations

import argparse
import ctypes as C

import numpy as np

from ._lib import YB_KMEANS_MAX_K, check, lib, ptr, stream_handle


def iou(box, clusters):
    """IoU of one (w, h) box against k (w, h) clusters, both anchored at the origin (host, float64)."""
    clusters = np.asarray(clusters)
    x = np.minimum(clusters[:, 0], box[0])
    y = np.minimum(clusters[:, 1], box[1])
    if np.count_nonzero(x == 0) > 0 or np.count_nonzero(y == 0) > 0:
        raise ValueError("Box has no area")
    inter = x * y
    return inter / (box[0] * box[1] + clusters[:, 0] * clusters[:, 1] - inter + 1e-10)


def translate_boxes(boxes):
    """[r, 4] (x_min, y_min, x_max, y_max) -> [r, 2] (|x_max - x_min|, |y_max - y_min|), in the input's dtype."""
    boxes = np.asarray(boxes)
    out = np.empty((boxes.shape[0], 2), dtype=boxes.dtype)
    out[:, 0] = np.abs(boxes[:, 2] - boxes[:, 0])
    out[:, 1] = np.abs(boxes[:, 3] - boxes[:, 1])
    return out


def parse_anno(annotation_path, target_size=None):
    """(w, h) of every box of a train.txt annotation file (`index path img_w img_h label x0 y0 x1 y1 ...` per line).
    With target_size = [W, H] the sizes are scaled as a letterbox resize to W x H scales them."""
    result = []
    with open(annotation_path, "r") as f:
        for line in f:
            s = line.strip().split(" ")
            img_w, img_h = int(s[2]), int(s[3])
            s = s[4:]
            for i in range(len(s) // 5):
                x_min, y_min, x_max, y_max = (float(v) for v in s[i * 5 + 1:i * 5 + 5])
                width, height = x_max - x_min, y_max - y_min
                if not (width > 0 and height > 0):
                    raise ValueError(f"parse_anno: box {s[i * 5:i * 5 + 5]} of {annotation_path} has no area")
                if target_size is not None:
                    ratio = min(target_size[0] / img_w, target_size[1] / img_h)
                    width *= ratio
                    height *= ratio
                result.append([width, height])
    return np.asarray(result)


def _device_pairs(a, what):
    """[r, 2] float64, finite and > 0, contiguous on the current CUDA device."""
    import torch
    if isinstance(a, torch.Tensor):
        t = a.detach().to(device="cuda", dtype=torch.float64).contiguous()
        if t.dim() != 2 or t.shape[1] != 2:
            raise ValueError(f"{what} must be [r, 2], got {tuple(t.shape)}")
        ok = bool(torch.all(torch.isfinite(t) & (t > 0))) if t.numel() else True
    else:
        h = np.ascontiguousarray(a, dtype=np.float64)
        if h.ndim != 2 or h.shape[1] != 2:
            raise ValueError(f"{what} must be [r, 2], got {h.shape}")
        ok = bool(np.all(np.isfinite(h) & (h > 0)))
        t = torch.from_numpy(h).cuda() if ok else None
    if not ok:
        raise ValueError(f"{what}: every width and height must be finite and > 0")
    return t


class KMeansSteps:
    """The device side of one clustering: the boxes, the [rows] assignment, the [k + 1] counts / changes and the
    workspace.  `assign`, `median` and `avg_iou` are one launch each (plus one small read for `assign`)."""

    def __init__(self, boxes, k):
        import torch
        k = int(k)
        if not 1 <= k <= YB_KMEANS_MAX_K:
            raise ValueError(f"kmeans: k = {k} outside [1, {YB_KMEANS_MAX_K}]")
        if len(boxes) < k:                                   # the ValueError np.random.choice would raise
            raise ValueError(f"kmeans: {len(boxes)} boxes < k = {k}: cannot take a larger sample than population")
        self.boxes = _device_pairs(boxes, "kmeans: boxes")
        self.rows, self.k = self.boxes.shape[0], k
        dev = self.boxes.device
        need = C.c_size_t()
        check(lib.yb_kmeans_workspace_bytes(self.rows, k, C.byref(need)), "yb_kmeans_workspace_bytes")
        self.ws = torch.empty((need.value,), dtype=torch.uint8, device=dev)
        self.assignment = torch.zeros((self.rows,), dtype=torch.int32, device=dev)
        self.result = torch.empty((k + 1,), dtype=torch.int32, device=dev)
        self.clusters = torch.empty((k, 2), dtype=torch.float64, device=dev)
        self._out = torch.empty((1,), dtype=torch.float64, device=dev)

    def set_clusters(self, clusters):
        c = _device_pairs(clusters, "kmeans: clusters")
        if c.shape[0] != self.k:
            raise ValueError(f"kmeans: {c.shape[0]} clusters, expected {self.k}")
        self.clusters.copy_(c)

    def assign(self):
        """Nearest cluster of every box, in place of the last assignment -> (counts [k], changes) on the host."""
        check(lib.yb_kmeans_assign(ptr(self.boxes), self.rows, ptr(self.clusters), self.k, ptr(self.assignment),
                                   ptr(self.assignment), ptr(self.result), ptr(self.ws), self.ws.numel(),
                                   stream_handle()), "yb_kmeans_assign")
        r = self.result.cpu().numpy()
        return r[:self.k], int(r[self.k])

    def median(self):
        """clusters[c] = np.median of the boxes assigned to c (NaN for an empty cluster)."""
        check(lib.yb_kmeans_median(ptr(self.boxes), self.rows, ptr(self.assignment), ptr(self.result), self.k,
                                   ptr(self.clusters), ptr(self.ws), self.ws.numel(), stream_handle()),
              "yb_kmeans_median")

    def avg_iou(self):
        check(lib.yb_kmeans_avg_iou(ptr(self.boxes), self.rows, ptr(self.clusters), self.k, ptr(self._out),
                                    ptr(self.ws), self.ws.numel(), stream_handle()), "yb_kmeans_avg_iou")
        return np.float64(self._out.item())

    def run(self, seed=None):
        """The reference's loop from a host draw of k distinct boxes; returns the iteration count."""
        import torch
        idx = np.random.RandomState(seed).choice(self.rows, self.k, replace=False)
        self.clusters.copy_(self.boxes[torch.from_numpy(idx).to(self.boxes.device)])
        self.assignment.zero_()                                  # get_kmeans.py:72
        it = 0
        while True:
            it += 1
            counts, changes = self.assign()
            if changes == 0:
                return it
            empty = np.flatnonzero(counts == 0)
            if empty.size:
                raise ValueError(f"kmeans: cluster {int(empty[0])} is empty at iteration {it} (the reference's loop "
                                 "would never return); try another seed or a smaller k")
            self.median()


def _check_dist(dist):
    if dist is not np.median:
        raise ValueError("kmeans: only dist=np.median is supported")


def kmeans(boxes, k, dist=np.median, seed=None):
    """k clusters of the [r, 2] boxes (numpy or CUDA tensor) -> numpy [k, 2] float64, as the reference's kmeans.
    seed=None draws the initial clusters from fresh entropy, as the reference does; numpy's global RNG is untouched."""
    _check_dist(dist)
    s = KMeansSteps(boxes, k)
    s.run(seed)
    return s.clusters.cpu().numpy()


def avg_iou(boxes, clusters):
    """Mean over the boxes of the best IoU with any cluster (numpy or CUDA tensor inputs) -> float64."""
    c = _device_pairs(clusters, "avg_iou: clusters")
    k = c.shape[0]
    if not 1 <= k <= YB_KMEANS_MAX_K:
        raise ValueError(f"avg_iou: k = {k} outside [1, {YB_KMEANS_MAX_K}]")
    b = _device_pairs(boxes, "avg_iou: boxes")
    if b.shape[0] < 1:
        raise ValueError("avg_iou: no boxes")
    import torch
    need = C.c_size_t()
    check(lib.yb_kmeans_workspace_bytes(b.shape[0], 1, C.byref(need)), "yb_kmeans_workspace_bytes")
    ws = torch.empty((need.value,), dtype=torch.uint8, device=b.device)
    out = torch.empty((1,), dtype=torch.float64, device=b.device)
    check(lib.yb_kmeans_avg_iou(ptr(b), b.shape[0], ptr(c), k, ptr(out), ptr(ws), ws.numel(), stream_handle()),
          "yb_kmeans_avg_iou")
    return np.float64(out.item())


def get_kmeans(anno, cluster_num=9, seed=None):
    """(anchors as a list of [w, h] ints sorted by area, average IoU of the float anchors), as the reference's."""
    s = KMeansSteps(anno, cluster_num)
    s.run(seed)
    ave_iou = s.avg_iou()
    anchors = s.clusters.cpu().numpy().astype("int").tolist()
    return sorted(anchors, key=lambda a: a[0] * a[1]), ave_iou


def main(argv=None):
    ap = argparse.ArgumentParser(description="k-means anchors of a train.txt annotation file")
    ap.add_argument("annotation_path")
    ap.add_argument("--target-size", type=int, nargs=2, default=[416, 416], metavar=("W", "H"),
                    help="cluster the sizes after a letterbox resize to W x H (default 416 416)")
    ap.add_argument("--original-size", action="store_true", help="cluster the sizes at the original image scale")
    ap.add_argument("--clusters", type=int, default=9)
    ap.add_argument("--seed", type=int, default=None)
    a = ap.parse_args(argv)
    boxes = parse_anno(a.annotation_path, target_size=None if a.original_size else a.target_size)
    anchors, ave_iou = get_kmeans(boxes, a.clusters, seed=a.seed)
    print("anchors are:")
    print(", ".join(f"{w},{h}" for w, h in anchors))
    print("the average iou is:")
    print(ave_iou)


if __name__ == "__main__":
    main()
