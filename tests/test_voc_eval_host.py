"""CPU tests of the device VOC evaluator's host side: pack_gt_rec, the C-ABI argument checks of yb_voc_match /
yb_voc_ap (which return before any device work), and the stable test oracle against the reference's golden rows."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import yolov3_oracle as O
from tests.synth import gen_eval_case
from tests.voc_ref import rows_from_nms, voc_eval_stable

NMS = dict(max_boxes=20, score_thresh=0.3, nms_thresh=0.45)


def test_pack_gt_rec_shapes_dtypes_padding():
    import torch
    from yolov3_tensorflow_b200.utils.eval_utils import pack_gt_rec
    gt = {7: [[1.5, 2.25, 30.0, 40.125, 3], [0.1, 0.2, 5.0, 6.0, 0]], 9: [], 11: [[10.0, 11.0, 12.0, 13.0, 79]]}
    b, l, c = pack_gt_rec(gt, [7, 9, 11, 12])
    assert (b.dtype, l.dtype, c.dtype) == (torch.float64, torch.int32, torch.int32)
    assert tuple(b.shape) == (4, 2, 4) and tuple(l.shape) == (4, 2) and tuple(c.shape) == (4,)
    assert c.tolist() == [2, 0, 1, 0]
    assert b[0].tolist() == [[1.5, 2.25, 30.0, 40.125], [0.1, 0.2, 5.0, 6.0]] and l[0].tolist() == [3, 0]
    assert b[2, 0].tolist() == [10.0, 11.0, 12.0, 13.0] and l[2, 0] == 79
    assert not b[1].any() and not b[2, 1].any() and not b[3].any()
    assert l[1].tolist() == [-1, -1] and l[2, 1] == -1 and l[3].tolist() == [-1, -1]
    b, l, c = pack_gt_rec(gt, [9], vmax=5)
    assert tuple(b.shape) == (1, 5, 4) and c.tolist() == [0]
    with pytest.raises(ValueError):
        pack_gt_rec(gt, [7], vmax=1)


def test_voc_abi_argument_checks():
    from yolov3_tensorflow_b200 import _lib
    lib = _lib.lib
    cc = C.c_void_p(16)            # never dereferenced: every call below fails its checks first
    args = lambda vmax, ncls: (cc, cc, cc, cc, 2, 10, cc, cc, cc, vmax, ncls, 0.5, cc, 0, 100, cc, None)
    assert lib.yb_voc_match(*args(_lib.YB_VOC_MAX_GT + 1, 80)) == -1
    assert b"vmax" in lib.yb_last_error_string()
    assert lib.yb_voc_match(*args(8, 0)) == -1
    assert b"num_classes" in lib.yb_last_error_string()
    assert lib.yb_voc_match(*args(8, 65536)) == -1
    bad_offset = (cc, cc, cc, cc, 2, 10, cc, cc, cc, 8, 80, 0.5, cc, 101, 100, cc, None)
    assert lib.yb_voc_match(*bad_offset) == -1
    n = C.c_size_t()
    assert lib.yb_voc_ap_workspace_bytes(1000, 0, C.byref(n)) == -1
    assert lib.yb_voc_ap_workspace_bytes(-1, 80, C.byref(n)) == -1
    assert lib.yb_voc_ap_workspace_bytes(1 << 20, 80, C.byref(n)) == 0 and n.value >= 2 * 8 << 20
    assert lib.yb_voc_ap(cc, 1 << 20, cc, 80, 0, cc, n.value - 1, cc, None) == -4
    assert b"workspace" in lib.yb_last_error_string()
    assert lib.yb_voc_ap(cc, 1 << 20, cc, 0, 0, cc, n.value, cc, None) == -1


def test_eleven_point_thresholds_are_k_tenths():
    """The device forms the 11-point thresholds as k * 0.1 in float64, which is what np.arange(0., 1.1, 0.1) holds."""
    assert np.array_equal(np.arange(0., 1.1, 0.1), np.asarray([k * 0.1 for k in range(11)]))


@pytest.mark.parametrize("tag", ["a", "b"])
def test_stable_oracle_matches_reference_golden(golden_dir, tag):
    g = np.load(os.path.join(golden_dir, "eval.npz"))
    seed, n, w, h, cn = (int(v) for v in g[f"ev_{tag}_cfg"])
    y_pred, _, gts = gen_eval_case(seed, n, w, h, cn)
    dets = []
    for i in range(n):
        b, s, l, _ = O.gpu_nms(y_pred[0][i:i + 1], (y_pred[1][i:i + 1] * y_pred[2][i:i + 1]).astype(np.float32), cn,
                               NMS["max_boxes"], NMS["score_thresh"], NMS["nms_thresh"])
        dets.append((b, s, l))
    rows = rows_from_nms([100 + i for i in range(n)], [d[0] for d in dets], [d[1] for d in dets], [d[2] for d in dets],
                         [len(d[2]) for d in dets])
    gt_dict = {100 + i: [[float(v) for v in b[:4]] + [int(l)] for b, l in zip(*gts[i])] for i in range(n)}
    for row in g[f"voc_{tag}"]:
        c, m07 = int(row[0]), bool(row[1])
        with np.errstate(divide="ignore", invalid="ignore"):
            r = voc_eval_stable(gt_dict, rows, c, 0.5, m07)
        assert np.array_equal(np.asarray([float(v) for v in r]), row[2:], equal_nan=True), (c, m07, r, row[2:])
