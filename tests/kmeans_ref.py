"""Vectorised numpy restatement of the reference's get_kmeans.py kmeans / avg_iou (CPU tests and the bench only), and
the seeded generators of the k-means test inputs.

Every step is the reference's arithmetic on whole arrays: the same float64 IoU expression (elementwise numpy ops round
exactly as the per-row ones do), np.argmin over 1 - IoU, np.median per cluster.  An empty cluster raises ValueError
where the reference would loop forever.  `pairwise_sum` models numpy's pairwise summation, so `avg_iou` is np.mean of
the per-box maxima without building the Python list."""
import numpy as np

PW_BLOCK = 128


# ---- inputs ---------------------------------------------------------------------------------------------------------
def gen_float_boxes(seed, n, lo=4.0, hi=416.0):
    """COCO-like box sizes: w and h log-uniform in [lo, hi]."""
    rng = np.random.default_rng(seed)
    return np.exp(rng.uniform(np.log(lo), np.log(hi), (n, 2)))


def gen_int_boxes(seed, n, hi=64):
    """Integer-valued sizes in [1, hi]^2: many equal values, ties and even-count medians."""
    return np.random.default_rng(seed).integers(1, hi + 1, (n, 2)).astype(np.float64)


def gen_xyxy(seed, n):
    """[n, 4] corner pairs in either order (translate_boxes takes |x1 - x0|, |y1 - y0|)."""
    return np.random.default_rng(seed).uniform(0.0, 500.0, (n, 4))


def gen_train_txt(seed, lines=6):
    """A train.txt in the reference's format: `index path img_w img_h (label x_min y_min x_max y_max)*` per line."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(lines):
        w, h = int(rng.integers(200, 1200)), int(rng.integers(200, 1200))
        parts = [str(i), f"/data/img_{i:04d}.jpg", str(w), str(h)]
        for _ in range(int(rng.integers(1, 6))):
            x0, y0 = rng.uniform(0, w - 20), rng.uniform(0, h - 20)
            x1, y1 = rng.uniform(x0 + 1, w), rng.uniform(y0 + 1, h)
            parts += [str(int(rng.integers(0, 80))), f"{x0:.2f}", f"{y0:.2f}", f"{x1:.2f}", f"{y1:.2f}"]
        out.append(" ".join(parts))
    return "\n".join(out) + "\n"


# ---- the algorithm --------------------------------------------------------------------------------------------------
def iou_matrix(boxes, clusters):
    """[r, k] IoU in the reference's operation order."""
    bw, bh = boxes[:, 0:1], boxes[:, 1:2]
    cw, ch = clusters[None, :, 0], clusters[None, :, 1]
    inter = np.minimum(cw, bw) * np.minimum(ch, bh)
    return inter / (bw * bh + cw * ch - inter + 1e-10)


def assign(boxes, clusters):
    return np.argmin(1 - iou_matrix(boxes, clusters), axis=1)


def medians(boxes, nearest, k, iteration=0):
    out = np.empty((k, 2))
    for c in range(k):
        sel = boxes[nearest == c]
        if sel.shape[0] == 0:
            raise ValueError(f"kmeans: cluster {c} is empty at iteration {iteration}")
        out[c] = np.median(sel, axis=0)
    return out


def initial_clusters(boxes, k, seed):
    return boxes[np.random.RandomState(seed).choice(boxes.shape[0], k, replace=False)]


def kmeans_trace(boxes, k, seed):
    """-> (final clusters, [assignment of every iteration], [clusters after every update])."""
    boxes = np.asarray(boxes, np.float64)
    clusters = initial_clusters(boxes, k, seed)
    last = np.zeros((boxes.shape[0],), np.int64)
    assigns, updates = [], []
    it = 0
    while True:
        it += 1
        nearest = assign(boxes, clusters)
        assigns.append(nearest)
        if (last == nearest).all():
            return clusters, assigns, updates
        clusters = medians(boxes, nearest, k, it)
        updates.append(clusters)
        last = nearest


def kmeans(boxes, k, seed):
    return kmeans_trace(boxes, k, seed)[0]


def _leaf(a, lo, n):
    if n < 8:
        r = 0.0
        for i in range(n):
            r += float(a[lo + i])
        return r
    body = n - n % 8
    r = a[lo:lo + 8].copy()
    for i in range(8, body, 8):
        r += a[lo + i:lo + i + 8]
    r = [float(v) for v in r]
    res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    for i in range(body, n):
        res += float(a[lo + i])
    return res


def pairwise_sum(a, lo=0, n=None):
    """numpy's pairwise summation of a contiguous float64 array (leaves of <= 128 with 8 accumulators)."""
    if n is None:
        a = np.ascontiguousarray(a, np.float64)
        n = a.shape[0]
    if n <= PW_BLOCK:
        return _leaf(a, lo, n)
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(a, lo, n2) + pairwise_sum(a, lo + n2, n - n2)


def avg_iou(boxes, clusters):
    m = np.max(iou_matrix(np.asarray(boxes, np.float64), np.asarray(clusters, np.float64)), axis=1)
    return np.float64(pairwise_sum(m) / m.shape[0])


def get_kmeans(boxes, k, seed):
    clusters = kmeans(boxes, k, seed)
    ave = avg_iou(boxes, clusters)
    return sorted(clusters.astype("int").tolist(), key=lambda a: a[0] * a[1]), ave
