"""CPU tests of the host-side mirror of the reference's utility functions (no GPU work): the numpy NMS variants
against the golden vectors produced by the reference's own code, anchor / class-name parsing, batch sharding and the
darknet weight file writer."""
import os

import numpy as np
import pytest

from oracle import yolov3_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _pkg():
    import yolov3_tensorflow_b200 as pkg
    return pkg


def test_cpu_and_py_nms_match_reference_golden(golden_dir):
    pkg = _pkg()
    g = np.load(os.path.join(golden_dir, "nms.npz"))
    cb, cs, cl = pkg.cpu_nms(g["boxes_in"][None], g["scores_in"][None], 6, max_boxes=20, score_thresh=0.3, iou_thresh=0.45)
    assert np.array_equal(cb, g["cpu_boxes"]) and np.array_equal(cs, g["cpu_scores"]) and np.array_equal(cl, g["cpu_labels"])
    assert list(pkg.py_nms(g["boxes_in"], g["scores_in"][:, 0], max_boxes=30, iou_thresh=0.5)) == list(g["py_keep"])


def test_cpu_nms_returns_none_triplet_without_candidates():
    pkg = _pkg()
    boxes = np.zeros((1, 5, 4), np.float32)
    scores = np.zeros((1, 5, 3), np.float32)
    assert pkg.cpu_nms(boxes, scores, 3, score_thresh=0.5) == (None, None, None)   # utils/nms_utils.py:118-119


def test_anchor_and_class_name_files():
    pkg = _pkg()
    data = os.path.join(ROOT, "yolov3_tensorflow_b200", "data")
    anchors = pkg.parse_anchors(os.path.join(data, "yolo_anchors.txt"))
    assert anchors.shape == (9, 2) and anchors.dtype == np.float32
    assert np.array_equal(anchors, np.asarray(O.COCO_ANCHORS, np.float32))
    names = pkg.read_class_names(os.path.join(data, "coco.names"))
    assert len(names) == 80 and names[0] == "person" and names[79] == "toothbrush"


def test_shard_batch_covers_the_batch_once():
    from yolov3_tensorflow_b200.parallel import shard_batch
    for n, world in ((256, 8), (64, 2), (64, 1)):
        spans = [shard_batch(n, r, world) for r in range(world)]
        assert spans[0][0] == 0 and spans[-1][1] == n
        assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
        assert len({hi - lo for lo, hi in spans}) == 1
    with pytest.raises(ValueError):          # equal shards only: every loss term is a mean over the local batch
        shard_batch(10, 0, 4)


def test_save_weights_writes_the_darknet_stream(tmp_path):
    from yolov3_tensorflow_b200.utils.misc_utils import save_weights
    params = O.make_params(80, seed=11, random_bn=True)
    path = tmp_path / "w.weights"
    save_weights(params, str(path), layout="HWIO")
    assert os.path.getsize(path) == 20 + 4 * 62_001_757
    back = O.load_darknet_weights(str(path), 80)          # the oracle's reader (utils/misc_utils.py:70-126 order)
    for a, b in zip(params, back):
        for k in a:
            assert np.array_equal(a[k], b[k]), k


# ------------------------------------------------------------------------- N1: LR schedules / optimizer selection
def _lr_args(**kw):
    import types
    base = dict(lr_type="exponential", learning_rate_init=1e-3, lr_decay_freq=400, lr_decay_factor=0.96, lr_lower_bound=1e-6,
                total_epoches=10, use_warm_up=True, warm_up_epoch=3, train_batch_num=100,
                pw_boundaries=[300.0, 500.0], pw_values=[1e-3, 3e-4, 1e-4])
    base.update(kw)
    return types.SimpleNamespace(**base)


def test_learning_rate_schedules_match_the_oracle_restatement():
    """utils/misc_utils.py:129-148 + warm-up train.py:93-99: the host-side schedule functions against the oracle's
    independent restatement (oracle.learning_rate) over all five lr types, with and without warm-up."""
    from oracle import yolov3_oracle as O
    from yolov3_tensorflow_b200.utils import misc_utils as M
    steps = [0, 1, 150, 299, 300, 301, 399, 400, 401, 799, 800, 1200, 2799, 2800, 5000]
    for kind in ("exponential", "cosine_decay", "cosine_decay_restart", "fixed", "piecewise"):
        for warm in (True, False):
            a = _lr_args(lr_type=kind, use_warm_up=warm)
            for s in steps:
                got, ref = M.learning_rate_at(a, s), O.learning_rate(a, s)
                assert abs(got - ref) <= 1e-12 + 1e-9 * abs(ref), (kind, warm, s, got, ref)
    assert M.learning_rate_at(_lr_args(), 150) == 1e-3 * 150 / 300                      # linear warm-up (train.py:95)
    assert M.config_learning_rate(_lr_args(lr_type="exponential"), 800) == max(1e-3 * 0.96 ** 2, 1e-6)
    assert M.config_learning_rate(_lr_args(lr_type="piecewise"), 300) == 1e-3 and M.config_learning_rate(_lr_args(lr_type="piecewise"), 300.5) == 3e-4
    with pytest.raises(ValueError, match="Unsupported learning rate type"):
        M.config_learning_rate(_lr_args(lr_type="poly"), 0)


def test_config_optimizer_and_tf_variable_names():
    from yolov3_tensorflow_b200.utils import misc_utils as M
    for name in ("momentum", "rmsprop", "adam", "sgd"):
        assert M.config_optimizer(name, 1e-3).name == name
    with pytest.raises(ValueError, match="Unsupported optimizer type"):
        M.config_optimizer("adagrad", 1e-3)                                                # utils/misc_utils.py:161
    names = M.tf_variable_names(80)
    assert len(names) == 72 * 5 + 3 * 2 == 366
    assert names[0][2] == "yolov3/darknet53_body/Conv/weights:0" and names[-1][2] == "yolov3/yolov3_head/Conv_22/biases:0"
    assert names[5][2] == "yolov3/darknet53_body/Conv_1/weights:0" and names[1][2] == "yolov3/darknet53_body/Conv/BatchNorm/gamma:0"


def _wgrad_desc(n, h, w, cin, cout, k, s):
    from yolov3_tensorflow_b200 import _lib as L
    return L.ConvDesc(n=n, h=h, w=w, cin=cin, cout=cout, ksize=k, stride=s, in_ld=cin, out_ld=cout, res_ld=0,
                      dtype=L.YB_F16, out_fp32=0, leaky=0, upsample2x=0)


def _wgrad_schedule(desc, sms=148, **opts):
    """yb_wgrad_schedule under the given YB_WGRAD_* options (restored afterwards)."""
    import ctypes as C
    from yolov3_tensorflow_b200 import _lib as L
    keys = ("YB_WGRAD_TP", "YB_WGRAD_EPI", "YB_WGRAD_SPLITS")
    info = L.WgradSchedule()
    try:
        for k in keys:
            L.set_option(k, opts.get(k))
        L.check(L.lib.yb_wgrad_schedule(C.byref(desc), sms, C.byref(info)), "yb_wgrad_schedule")
    finally:
        for k in keys:
            L.set_option(k, None)
    return info


# (n, h, w, cin, cout, k, s) -> (64-pixel blocks, tiles): the training step's layers at batch 32 @416 and a few more
WGRAD_PLAN_DESCS = {
    (32, 208, 208, 64, 32, 1, 1): (21632, 1),
    (32, 104, 104, 64, 128, 3, 1): (5408, 3),
    (32, 52, 52, 128, 128, 3, 1): (1352, 6),
    (32, 26, 26, 256, 256, 3, 1): (338, 24),
    (32, 13, 13, 512, 512, 3, 1): (85, 96),
    (32, 13, 13, 1024, 512, 1, 1): (85, 32),
    (32, 52, 52, 256, 128, 1, 1): (1352, 2),
    (1, 8, 8, 64, 64, 1, 1): (1, 1),
    (1, 20, 21, 3200, 2048, 1, 1): (7, 400),
    (1, 250, 256, 4768, 128, 1, 1): (1000, 149),
    (1, 64, 64, 64, 64, 1, 1): (64, 1),
}


def test_wgrad_schedule_one_wave_and_every_block_once():
    """Host logic of yb_conv2d_wgrad (csrc/conv_wgrad.cu: yb_wgrad_schedule): the split-K count minimises
    waves x (pixel blocks per CTA + epilogue); every 64-pixel block is covered exactly once, no split is empty."""
    want = {(21632, 1): (148, 147), (5408, 3): (49, 111), (1352, 6): (24, 57), (338, 24): (6, 57), (85, 96): (1, 85),
            (85, 32): (4, 22), (1352, 2): (72, 19)}
    for shape, (num_kb, tiles) in WGRAD_PLAN_DESCS.items():
        i = _wgrad_schedule(_wgrad_desc(*shape))
        assert (i.num_kb, i.tiles) == (num_kb, tiles), shape
        assert (i.grid_x, i.grid_y * i.grid_z) == (i.splits, i.tiles)
        if (num_kb, tiles) in want:
            assert (i.splits, i.kb_per_split) == want[(num_kb, tiles)], (shape, i.splits, i.kb_per_split)
        s, k = i.splits, i.kb_per_split
        assert s >= 1 and (s - 1) * k < num_kb <= s * k
        if tiles <= 148 and num_kb >= 148 // tiles:
            assert tiles * s <= 148                 # one wave of one-CTA-per-SM blocks whenever the work allows it
    # ignoring the epilogue cost (the first version's behaviour) splits further
    d = _wgrad_desc(32, 26, 26, 256, 256, 3, 1)
    assert _wgrad_schedule(d, YB_WGRAD_EPI="0").splits > _wgrad_schedule(d).splits
    with pytest.raises(Exception):
        _wgrad_schedule(_wgrad_desc(1, 8, 8, 48, 64, 1, 1))      # cin not a multiple of 32
    with pytest.raises(Exception):
        _wgrad_schedule(_wgrad_desc(1, 8, 8, 64, 64, 1, 1), sms=0)


def test_wgrad_schedule_kernel_choice_and_ring_depth():
    """bnw / tp / stages of the five kernel instantiations: (128, 1) for 1x1 with cin % 128 == 0, one kernel row of
    taps for 3x3 unless YB_WGRAD_TP=1, and the ring depth that 192 KB of stages allows (at most 8)."""
    cases = [((1, 16, 16, 256, 64, 1, 1), {}, (128, 1, 6)),
             ((1, 16, 16, 64, 64, 1, 1), {}, (64, 1, 8)),
             ((1, 16, 16, 96, 64, 1, 1), {}, (32, 1, 8)),
             ((1, 16, 16, 128, 64, 3, 1), {}, (64, 3, 4)),
             ((1, 16, 16, 32, 64, 3, 2), {}, (32, 3, 6)),
             ((1, 16, 16, 128, 64, 3, 1), {"YB_WGRAD_TP": "1"}, (64, 1, 8)),
             ((1, 16, 16, 32, 64, 3, 1), {"YB_WGRAD_TP": "1"}, (32, 1, 8))]
    for shape, opts, want in cases:
        i = _wgrad_schedule(_wgrad_desc(*shape), **opts)
        assert (i.bnw, i.tp, i.stages) == want, (shape, opts)
        n, h, w, cin, cout, k, s = shape
        assert i.grid_y == k * k // i.tp * (cin // i.bnw) and i.grid_z == -(-cout // 128)


def test_wgrad_schedule_forced_splits_clamp():
    """YB_WGRAD_SPLITS=N forces the split count, clamped to [1, num_kb]: kb_per_split = ceil(num_kb / N) and the
    effective count is ceil(num_kb / kb_per_split)."""
    d = _wgrad_desc(2, 20, 16, 64, 128, 3, 1)           # 640 pixels = 10 blocks
    assert _wgrad_schedule(d).num_kb == 10
    for forced, (kbs, splits) in {"1": (10, 1), "3": (4, 3), "4": (3, 4), "6": (2, 5), "7": (2, 5), "9": (2, 5),
                                  "10": (1, 10), "11": (1, 10), "100000": (1, 10), "0": (10, 1),
                                  "-3": (10, 1)}.items():
        i = _wgrad_schedule(d, YB_WGRAD_SPLITS=forced)
        assert (i.kb_per_split, i.splits, i.grid_x) == (kbs, splits, splits), (forced, i.kb_per_split, i.splits)
        assert (i.splits - 1) * i.kb_per_split < i.num_kb <= i.splits * i.kb_per_split
    # the forced count overrides the cost model (and the SM count) but not the tile decomposition
    big = _wgrad_desc(32, 208, 208, 64, 32, 1, 1)
    i = _wgrad_schedule(big, sms=4, YB_WGRAD_SPLITS="1000")
    assert (i.splits, i.kb_per_split, i.tiles) == (984, 22, 1)       # 21632 blocks: ceil(21632 / 1000) = 22 per split
    assert _wgrad_schedule(big, YB_WGRAD_SPLITS="1000", YB_WGRAD_TP="1").tiles == 1


def test_conv3x3_halo_supported_grid():
    """yb_conv3x3_halo_supported (csrc/conv_halo.cu): 3x3 convs, stride 1 | 2, cin 32 | 64 and cout 64 | 128 except
    64 -> 128 at stride 2 (its weights and one parity-plane stage exceed shared memory), fp16 / bf16 operands, a 16-bit
    non-upsampled output, an output width (w / stride) that is a multiple of 8 and leading dimensions that are multiples
    of 8."""
    import ctypes as C
    import itertools
    from yolov3_tensorflow_b200 import _lib as L
    got, want = set(), set()
    for cin, cout, s, wo, dt, f32, up, bad_ld in itertools.product((32, 64, 96), (32, 64, 128), (1, 2), (16, 24, 20),
                                                                   (L.YB_F16, L.YB_BF16, L.YB_E4M3), (0, 1), (0, 1),
                                                                   (None, "in", "out")):
        d = L.ConvDesc(n=2, h=16 * s, w=wo * s, cin=cin, cout=cout, ksize=3, stride=s,
                       in_ld=cin + (4 if bad_ld == "in" else 0), out_ld=cout + (4 if bad_ld == "out" else 0), res_ld=0,
                       dtype=dt, out_fp32=f32, leaky=1, upsample2x=up)
        key = (cin, cout, s, wo, dt, f32, up, bad_ld)
        if L.lib.yb_conv3x3_halo_supported(C.byref(d)):
            got.add(key)
        if (cin in (32, 64) and cout in (64, 128) and (cin, cout, s) != (64, 128, 2) and wo % 8 == 0
                and dt in (L.YB_F16, L.YB_BF16) and not f32 and not up and bad_ld is None):
            want.add(key)
    assert got == want
    assert len(want) == 7 * 2 * 2       # 7 (cin, cout, stride) kernels x 2 widths x 2 types
