"""Device k-means anchors (yolov3_tensorflow_b200.get_kmeans: yb_kmeans_assign / yb_kmeans_median / yb_kmeans_avg_iou)
against the reference's golden vectors and the numpy restatement (tests/kmeans_ref.py).  Equal means bit for bit:
every assignment, every cluster value, avg_iou and the anchors."""
import os

import numpy as np
import pytest

from tests import kmeans_ref as K

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kmeans.npz")
TAGS = ("a", "b1", "b2", "b6", "b9", "b12", "c")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def golden_case(g, tag):
    gen, bseed, rows, k, iseed = (int(v) for v in g[f"{tag}_cfg"])
    if gen == 0:
        boxes = K.gen_float_boxes(bseed, rows)
    elif gen == 1:
        boxes = K.gen_int_boxes(bseed, rows)
    else:
        boxes = np.tile(np.array([[20.0, 30.0]]), (rows, 1))
    return boxes, k, iseed


def same_bits(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def G():
    from yolov3_tensorflow_b200 import get_kmeans
    return get_kmeans


def stepped(boxes, k, seed):
    """Drive the three entry points one iteration at a time; check counts and the assignment range on the way.
    -> (assignment of every iteration, clusters after every update, final avg_iou)."""
    s = G().KMeansSteps(boxes, k)
    s.set_clusters(K.initial_clusters(boxes, k, seed))
    assigns, updates = [], []
    while True:
        counts, changes = s.assign()
        a = s.assignment.cpu().numpy()
        assert counts.sum() == boxes.shape[0] and a.min() >= 0 and a.max() < k
        assert np.array_equal(counts, np.bincount(a, minlength=k))
        assigns.append(a)
        if changes == 0:
            return assigns, updates, s.avg_iou()
        prev = assigns[-2] if len(assigns) > 1 else np.zeros_like(a)
        assert changes == int(np.count_nonzero(a != prev))
        s.median()
        updates.append(s.clusters.cpu().numpy())


@pytest.mark.parametrize("tag", TAGS)
def test_golden_kmeans_avg_iou_get_kmeans(g, tag):
    boxes, k, seed = golden_case(g, tag)
    assert same_bits(G().kmeans(boxes, k, seed=seed), g[f"{tag}_clusters"])
    assert same_bits(G().avg_iou(boxes, g[f"{tag}_clusters"]), g[f"{tag}_avg_iou"])
    anchors, ave = G().get_kmeans(boxes, k, seed=seed)
    assert anchors == g[f"{tag}_anchors"].tolist() and same_bits(ave, g[f"{tag}_ave_iou"])


@pytest.mark.parametrize("tag", TAGS)
def test_golden_stepwise(g, tag):
    boxes, k, seed = golden_case(g, tag)
    assigns, updates, ave = stepped(boxes, k, seed)
    ref = g[f"{tag}_assign"]
    assert len(assigns) == ref.shape[0]
    for it, (a, r) in enumerate(zip(assigns, ref)):
        assert np.array_equal(a, r), f"iteration {it + 1}"
    _, ref_assigns, ref_updates = K.kmeans_trace(boxes, k, seed)
    assert len(updates) == len(ref_updates)
    for it, (c, r) in enumerate(zip(updates, ref_updates)):
        assert same_bits(c, r), f"update {it + 1}"
    assert same_bits(ave, g[f"{tag}_avg_iou"])


def test_cuda_tensor_input_equals_numpy(g):
    import torch
    boxes, k, seed = golden_case(g, "a")
    t = torch.from_numpy(boxes).cuda()
    assert same_bits(G().kmeans(t, k, seed=seed), g["a_clusters"])
    assert same_bits(G().avg_iou(t, torch.from_numpy(g["a_clusters"]).cuda()), g["a_avg_iou"])
    assert same_bits(G().kmeans(t.float(), k, seed=seed), K.kmeans(boxes.astype(np.float32).astype(np.float64), k, seed))


def test_large_float_boxes_k9():
    boxes = K.gen_float_boxes(41, 1_000_000)
    clusters, assigns, _ = K.kmeans_trace(boxes, 9, 200)
    s = G().KMeansSteps(boxes, 9)
    assert s.run(200) == len(assigns)
    assert np.array_equal(s.assignment.cpu().numpy(), assigns[-1])
    assert same_bits(s.clusters.cpu().numpy(), clusters)
    assert same_bits(s.avg_iou(), K.avg_iou(boxes, clusters))


@pytest.mark.parametrize("k", [1, 2, 6, 9, 32])
def test_large_integer_boxes(k):
    boxes = K.gen_int_boxes(40, 200_000)
    clusters, assigns, updates = K.kmeans_trace(boxes, k, 100)
    got, got_updates, ave = stepped(boxes, k, 100)
    assert len(got) == len(assigns) and all(np.array_equal(a, b) for a, b in zip(got, assigns))
    assert all(same_bits(a, b) for a, b in zip(got_updates, updates))
    assert same_bits(ave, K.avg_iou(boxes, clusters))
    anchors, ave2 = G().get_kmeans(boxes, k, seed=100)
    assert (anchors, ave2) == K.get_kmeans(boxes, k, 100) and same_bits(ave2, ave)


@pytest.mark.parametrize("n", [1, 7, 8, 9, 127, 128, 129, 8192, 8193, 10 ** 6 + 3])
def test_avg_iou_tree_boundaries(n):
    boxes = K.gen_float_boxes(n + 1, n)
    clusters = K.gen_float_boxes(7, 9)
    assert same_bits(G().avg_iou(boxes, clusters), K.avg_iou(boxes, clusters))
    if n <= 8193:
        assert same_bits(G().avg_iou(boxes, clusters), np.mean([np.max(G().iou(b, clusters)) for b in boxes]))


def test_empty_cluster_raises_and_median_gives_nan():
    boxes = np.array([[10.0, 10.0], [10.0, 10.0], [200.0, 200.0]])
    with pytest.raises(ValueError, match="empty at iteration 1"):
        G().kmeans(boxes, 3, seed=0)
    s = G().KMeansSteps(boxes, 3)
    s.set_clusters(boxes)                       # clusters 0 and 1 are equal: ties go to 0, so 1 gets no box
    counts, changes = s.assign()
    assert counts.tolist() == [2, 0, 1] and changes == 1
    s.median()
    c = s.clusters.cpu().numpy()
    assert np.isnan(c[1]).all() and c[0].tolist() == [10.0, 10.0] and c[2].tolist() == [200.0, 200.0]


def test_bad_inputs_raise():
    import torch
    boxes = K.gen_float_boxes(3, 100)
    for bad in (0.0, -2.0, np.nan, np.inf):
        b = boxes.copy()
        b[17, 0] = bad
        for arg in (b, torch.from_numpy(b).cuda()):
            with pytest.raises(ValueError, match="finite and > 0"):
                G().kmeans(arg, 9)
            with pytest.raises(ValueError, match="finite and > 0"):
                G().avg_iou(arg, boxes[:9])
    with pytest.raises(ValueError):
        G().kmeans(boxes[:5], 9)
    with pytest.raises(ValueError, match="outside"):
        G().kmeans(boxes, 33)
    with pytest.raises(ValueError, match="np.median"):
        G().kmeans(boxes, 9, dist=np.mean)
    with pytest.raises(ValueError, match="outside"):
        G().avg_iou(boxes, np.ones((33, 2)))


def test_cli_prints_reference_lines(tmp_path, capsys):
    path = tmp_path / "train.txt"
    path.write_text(K.gen_train_txt(11, lines=40))
    G().main([str(path), "--clusters", "4", "--seed", "3"])
    out = capsys.readouterr().out.splitlines()
    boxes = G().parse_anno(str(path), target_size=[416, 416])
    anchors, ave = K.get_kmeans(boxes, 4, 3)
    assert out == ["anchors are:", ", ".join(f"{w},{h}" for w, h in anchors), "the average iou is:", str(ave)]
