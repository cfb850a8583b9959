"""CPU tests of k-means anchors: the numpy restatement (tests/kmeans_ref.py) against the reference's golden vectors
iteration by iteration, the pairwise-sum model against np.mean, the host-side parse_anno / translate_boxes / iou of
yolov3_tensorflow_b200.get_kmeans, and the C-ABI argument checks (which return before any device work)."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import kmeans_ref as K

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kmeans.npz")
TAGS = ("a", "b1", "b2", "b6", "b9", "b12", "c")


def golden_case(g, tag):
    gen, bseed, rows, k, iseed = (int(v) for v in g[f"{tag}_cfg"])
    if gen == 0:
        boxes = K.gen_float_boxes(bseed, rows)
    elif gen == 1:
        boxes = K.gen_int_boxes(bseed, rows)
    else:
        boxes = np.tile(np.array([[20.0, 30.0]]), (rows, 1))
    return boxes, k, iseed


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def same_bits(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


@pytest.mark.parametrize("tag", TAGS)
def test_restatement_equals_reference(g, tag):
    boxes, k, seed = golden_case(g, tag)
    clusters, assigns, _ = K.kmeans_trace(boxes, k, seed)
    ref_assigns = g[f"{tag}_assign"]
    assert len(assigns) == ref_assigns.shape[0]
    for it, (a, r) in enumerate(zip(assigns, ref_assigns)):
        assert np.array_equal(a, r), f"iteration {it + 1}"
    assert same_bits(clusters, g[f"{tag}_clusters"])
    assert same_bits(K.avg_iou(boxes, clusters), g[f"{tag}_avg_iou"])
    anchors, ave = K.get_kmeans(boxes, k, seed)
    assert anchors == g[f"{tag}_anchors"].tolist() and same_bits(ave, g[f"{tag}_ave_iou"])


def test_first_iteration_stop_returns_initial_clusters(g):
    boxes, k, seed = golden_case(g, "c")
    assert g["c_assign"].shape[0] == 1 and not g["c_assign"].any()
    assert same_bits(K.kmeans(boxes, k, seed), K.initial_clusters(boxes, k, seed))


@pytest.mark.parametrize("n", [1, 7, 8, 9, 127, 128, 129, 8192, 8193, 10 ** 6 + 3])
def test_pairwise_model_equals_np_mean(n):
    rng = np.random.default_rng(n)
    a = rng.random(n) * 10.0 ** rng.uniform(-4, 4, n)
    assert same_bits(K.pairwise_sum(a) / n, np.mean(list(a)))
    assert same_bits(K.pairwise_sum(a) / n, np.mean(a))


def test_empty_cluster_raises():
    boxes = np.array([[10.0, 10.0], [10.0, 10.0], [11.0, 11.0], [200.0, 200.0]])
    # clusters: boxes 0 and 1 are the same, so after the first assignment cluster 1 has no box
    clusters = boxes[[0, 1, 3]]
    nearest = K.assign(boxes, clusters)
    assert nearest.tolist() == [0, 0, 0, 2]
    with pytest.raises(ValueError, match="cluster 1 is empty at iteration 1"):
        K.medians(boxes, nearest, 3, 1)


def test_parse_anno_and_translate_boxes(g, tmp_path):
    from yolov3_tensorflow_b200 import get_kmeans as G
    path = tmp_path / "train.txt"
    path.write_text(K.gen_train_txt(int(g["anno_seed"])))
    assert same_bits(G.parse_anno(str(path), target_size=[416, 416]), g["anno_416"])
    assert same_bits(G.parse_anno(str(path), target_size=None), g["anno_none"])
    assert same_bits(G.translate_boxes(K.gen_xyxy(int(g["xyxy_seed"]), 40)), g["translated"])
    assert same_bits(G.iou(g["iou_box"], K.gen_float_boxes(3, 9)), g["iou"])
    with pytest.raises(ValueError, match="no area"):
        G.iou([0.0, 3.0], np.array([[1.0, 2.0]]))
    bad = tmp_path / "bad.txt"
    bad.write_text("0 a.jpg 100 100 3 10 10 10 20\n")
    with pytest.raises(ValueError, match="no area"):
        G.parse_anno(str(bad))


def test_kmeans_abi_argument_checks():
    from yolov3_tensorflow_b200 import _lib
    lib = _lib.lib
    cc = C.c_void_p(256)           # never dereferenced: every call below fails its checks first
    n = C.c_size_t()
    assert lib.yb_kmeans_workspace_bytes(1000, 0, C.byref(n)) == -1
    assert b"k 0" in lib.yb_last_error_string()
    assert lib.yb_kmeans_workspace_bytes(1000, _lib.YB_KMEANS_MAX_K + 1, C.byref(n)) == -1
    assert lib.yb_kmeans_workspace_bytes(8, 9, C.byref(n)) == -1
    assert b"rows" in lib.yb_last_error_string()
    assert lib.yb_kmeans_workspace_bytes(1 << 20, 9, C.byref(n)) == 0 and n.value >= 8 << 20
    need = n.value
    for k, rows in ((0, 100), (33, 100), (9, 8)):
        assert lib.yb_kmeans_assign(cc, rows, cc, k, cc, cc, cc, cc, 1 << 30, None) == -1
        assert lib.yb_kmeans_median(cc, rows, cc, cc, k, cc, cc, 1 << 30, None) == -1
    assert lib.yb_kmeans_assign(cc, 1 << 20, cc, 9, cc, cc, cc, cc, need - 1, None) == -4
    assert lib.yb_kmeans_median(cc, 1 << 20, cc, cc, 9, cc, cc, need - 1, None) == -4
    assert b"workspace" in lib.yb_last_error_string()
    assert lib.yb_kmeans_assign(C.c_void_p(264), 1 << 20, cc, 9, cc, cc, cc, cc, need, None) == -1
    assert b"aligned" in lib.yb_last_error_string()
    assert lib.yb_kmeans_avg_iou(cc, 0, cc, 9, cc, cc, 1 << 30, None) == -1
    assert lib.yb_kmeans_avg_iou(cc, 100, cc, 33, cc, cc, 1 << 30, None) == -1
    assert lib.yb_kmeans_avg_iou(cc, 5, cc, 9, cc, cc, 16, None) == -4              # rows < k is fine for avg_iou


def test_python_checks_need_no_device():
    from yolov3_tensorflow_b200 import get_kmeans as G
    boxes = K.gen_float_boxes(0, 20)
    with pytest.raises(ValueError, match="np.median"):
        G.kmeans(boxes, 3, dist=np.mean)
    with pytest.raises(ValueError, match="outside"):
        G.kmeans(boxes, 33)
    with pytest.raises(ValueError, match="outside"):
        G.kmeans(boxes, 0)
    for bad in (0.0, -1.0, np.nan, np.inf):
        b = boxes.copy()
        b[3, 1] = bad
        with pytest.raises(ValueError, match="finite and > 0"):
            G.kmeans(b, 3)
    with pytest.raises(ValueError, match="boxes < k"):
        G.kmeans(boxes[:2], 3)
    with pytest.raises(ValueError, match=r"\[r, 2\]"):
        G.avg_iou(np.ones((4, 2)), np.ones((2, 3)))
    with pytest.raises(ValueError, match="finite and > 0"):
        G.avg_iou(np.ones((4, 2)), -np.ones((2, 2)))
