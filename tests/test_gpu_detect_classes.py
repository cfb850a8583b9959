"""GPU tests of the fused detection heads at every class count from 1 to 80: model.detect_raw (decode and score filter
inside the head epilogues, then the greedy selection) must be bit-identical to forward() -> predict_scores() ->
batched_nms_raw() in all six arrays, in fp16, bf16 and on quantize_fp8 models, and every such plan must run the fused
path (yb_net_detect_supported) on the head tile width yb_net_layer_schedule reports.  The counts cover each tile-width
boundary (64 | 128 | 256 columns for 3 (5 + C)), the 256-column tiles over 192 rows of weights (C 38-59), and 3 (5 + C)
on and off a 32-column staging-chunk boundary.  Weights are cfg-2-like (heads x 8, conf bias -2) so candidates exist."""
import ctypes as C
import functools

import pytest
import torch

from oracle import yolov3_oracle as O
from tests.synth import gen_inputs

pytestmark = pytest.mark.gpu

CLASSES = (1, 2, 3, 5, 9, 16, 17, 20, 27, 37, 38, 43, 59, 60, 79, 80)
SIZES = ((416, 416), (288, 480))
SETTINGS = ((0.3, 200), (0.01, 400))     # (score_thresh, max_boxes): test_single_image.py's and the evaluation's
NMS_IOU = 0.45
BATCH = 2


def _tile(cn):
    """The fused head's n-tile: the narrowest wgmma width that holds all 3 (5 + C) columns."""
    cols = 3 * (5 + cn)
    return 64 if cols <= 64 else (128 if cols <= 128 else 256)


@functools.lru_cache(maxsize=1)
def _params(cn):
    return O.make_params(cn, seed=300 + cn, random_bn=True, det_scale=8.0, conf_bias=-2.0)


def _model(cn, dtype):
    import yolov3_tensorflow_b200 as pkg
    m = pkg.yolov3(cn, O.COCO_ANCHORS, dtype=dtype)
    m.set_params(_params(cn), "HWIO")
    return m


def _head_tiles(plan):
    """det_block_n of the three detection heads (yb_net_layer_schedule on a 132-SM device)."""
    from yolov3_tensorflow_b200 import _lib as L
    tiles = []
    for i in range(plan.num_layers):
        if plan.layer_info(i).has_bn:
            continue
        s = L.LayerSchedule()
        L.check(L.lib.yb_net_layer_schedule(plan.handle, i, 132, C.byref(s)), "yb_net_layer_schedule")
        tiles.append(s.det_block_n)
    return tiles


def _assert_same(unfused_boxes, unfused, fused, what):
    """fused = detect_raw's (boxes, out_boxes, out_scores, out_labels, out_indices, counts); unfused = batched_nms_raw's
    (out_boxes, out_scores, out_labels, out_indices, counts).  Slots past an image's count are unspecified."""
    assert torch.equal(fused[0], unfused_boxes), f"{what}: decoded boxes differ"
    assert torch.equal(fused[5], unfused[4]), f"{what}: counts {fused[5].tolist()} != {unfused[4].tolist()}"
    counts = unfused[4].tolist()
    assert sum(counts) > 0, f"{what}: no detections, the comparison would be empty"
    for i, k in enumerate(counts):
        for name, a, b in zip(("out_boxes", "out_scores", "out_labels", "out_indices"), unfused[:4], fused[1:5]):
            assert torch.equal(a[i, :k], b[i, :k]), f"{what}: {name} of image {i} differ"


def _check_model(m, cn, what, sizes=SIZES):
    from yolov3_tensorflow_b200 import _lib as L
    from yolov3_tensorflow_b200.utils.nms_utils import batched_nms_raw
    for h, w in sizes:
        x = torch.from_numpy(gen_inputs(cn * 7 + h, BATCH, h, w)).cuda()
        boxes, scores = m.predict_scores(m.forward(x))
        plan = m._last_plan
        assert L.lib.yb_net_detect_supported(plan.handle) == 1, f"{what}: no fused heads for {cn} classes"
        assert _head_tiles(plan) == [_tile(cn)] * 3
        for thr, mb in SETTINGS:
            unfused = batched_nms_raw(boxes, scores, cn, mb, thr, NMS_IOU)
            fused = m.detect_raw(x, mb, thr, NMS_IOU)
            _assert_same(boxes, unfused, fused, f"{what} {h}x{w} thr {thr} max_boxes {mb}")


@pytest.mark.parametrize("cn,dtype", [(cn, dt) for cn in CLASSES for dt in ("fp16", "bf16")])
def test_detect_fused_equals_three_calls(cn, dtype):
    _check_model(_model(cn, dtype), cn, f"{cn} classes {dtype}")


@pytest.mark.parametrize("cn", (1, 16, 17, 43, 80))
def test_detect_fused_equals_three_calls_fp8(cn):
    """A quantize_fp8 model takes the fused heads at the same class counts, with the same bits as its own three calls."""
    calib = torch.from_numpy(gen_inputs(900 + cn, BATCH, 416, 416)).cuda()
    qm = _model(cn, "fp16").quantize_fp8(calib)
    _check_model(qm, cn, f"{cn} classes e4m3", sizes=((416, 416),))


def test_more_than_80_classes_keep_three_calls():
    """81 classes do not fit one 256-column tile: no fused heads, and detect_raw returns the three calls' result."""
    from yolov3_tensorflow_b200 import _lib as L
    from yolov3_tensorflow_b200.utils.nms_utils import batched_nms_raw
    cn = 81
    m = _model(cn, "fp16")
    x = torch.from_numpy(gen_inputs(81, BATCH, 416, 416)).cuda()
    boxes, scores = m.predict_scores(m.forward(x))
    plan = m._last_plan
    assert L.lib.yb_net_detect_supported(plan.handle) == 0
    assert _head_tiles(plan) == [0, 0, 0]
    for thr, mb in SETTINGS:
        _assert_same(boxes, batched_nms_raw(boxes, scores, cn, mb, thr, NMS_IOU), m.detect_raw(x, mb, thr, NMS_IOU),
                     f"81 classes thr {thr}")


def test_custom_count_graphed_and_phases():
    """At a custom class count (43: a 256-column tile over 192 weight rows) detect_graphed returns detect_raw's bits, and
    detect_raw split into phases 1, 2, 4 (the benchmarks' brackets, reusing one result tuple) equals phases 7."""
    cn = 43
    m = _model(cn, "fp16")
    for seed in (1, 2):
        x = torch.from_numpy(gen_inputs(seed, 1, 288, 480)).cuda()
        e = [t.clone() for t in m.detect_raw(x, 200, 0.3, NMS_IOU)]
        g = m.detect_graphed(x, 200, 0.3, NMS_IOU)
        k = int(e[5][0])
        assert k > 0 and int(g[5][0]) == k
        assert torch.equal(g[0], e[0])
        for a, b in zip(g[1:5], e[1:5]):
            assert torch.equal(a[0, :k], b[0, :k])
    x = torch.from_numpy(gen_inputs(3, BATCH, 416, 416)).cuda()
    whole = [t.clone() for t in m.detect_raw(x, 200, 0.3, NMS_IOU)]
    res = m.detect_raw(x, 200, 0.01, NMS_IOU)                  # a different result first: every phase must overwrite it
    for ph in (1, 2, 4):
        m.detect_raw(x, 200, 0.3, NMS_IOU, phases=ph, out=res)
    assert torch.equal(res[0], whole[0]) and torch.equal(res[5], whole[5])
    for i, k in enumerate(whole[5].tolist()):
        for a, b in zip(res[1:5], whole[1:5]):
            assert torch.equal(a[i, :k], b[i, :k])
