"""Device VOC evaluation (utils.eval_utils.VOCEvaluator: yb_voc_match + yb_voc_ap) against the reference's golden rows,
the stable voc_eval oracle (tests/voc_ref.py) and, for sets too large for it, TP flags known by construction.
Equal means npos, nd, rec, prec and the 11-point AP bit-exact (nan-aware), the area AP within 1e-12."""
import os

import numpy as np
import pytest

from tests.voc_ref import assert_voc_equal, rows_from_nms, voc_eval_stable_all, voc_from_flags

pytestmark = pytest.mark.gpu


def _cuda(*arrays):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def _evaluate(batches, num_classes):
    """batches: [(ob, os, ol, cnt, gb, gl, gc)] numpy -> (area result, 11-point result)."""
    from yolov3_tensorflow_b200.utils.eval_utils import VOCEvaluator
    ev = VOCEvaluator(num_classes)
    for ob, os_, ol, cnt, gb, gl, gc in batches:
        ev.add_batch(*_cuda(ob, os_, ol, cnt, gb, gl, gc))
    return ev.result(False), ev.result(True)


def _oracle(batches, num_classes):
    rows, gt_dict, img = [], {}, 0
    for ob, os_, ol, cnt, gb, gl, gc in batches:
        ids = list(range(img, img + len(cnt)))
        rows += rows_from_nms(ids, ob, os_, ol, cnt)
        for i, k in zip(ids, gc):
            gt_dict[i] = [[float(v) for v in gb[i - img, j]] + [int(gl[i - img, j])] for j in range(int(k))]
        img += len(cnt)
    return voc_eval_stable_all(gt_dict, rows, num_classes)


def _check(batches, num_classes):
    area, p11 = _evaluate(batches, num_classes)
    want_area, want_11 = _oracle(batches, num_classes)
    assert_voc_equal(area, want_area)
    assert_voc_equal(p11, want_11, use_07_metric=True)
    return area, p11


def _layout(dets, gts, num_classes, vmax=None, cap=None):
    """Per-image lists -> the fixed [n, cap] NMS layout.  dets[i] = (boxes [K,4], scores [K], labels [K]) are put in NMS
    order (class ascending, score descending, stable); gts[i] = (boxes [V,4] float64, labels [V])."""
    n = len(dets)
    cap = cap or max(1, max(len(d[1]) for d in dets))
    vmax = vmax or max(1, max(len(g[1]) for g in gts))
    rng = np.random.default_rng(0)
    ob = rng.uniform(-5, 5, (n, cap, 4)).astype(np.float32)            # garbage past counts must be ignored
    os_ = rng.random((n, cap), dtype=np.float32)
    ol = rng.integers(0, num_classes, (n, cap)).astype(np.int32)
    cnt = np.zeros(n, np.int32)
    gb = np.zeros((n, vmax, 4), np.float64)
    gl = np.full((n, vmax), -1, np.int32)
    gc = np.zeros(n, np.int32)
    for i, ((b, s, l), (g, gl_i)) in enumerate(zip(dets, gts)):
        s = np.asarray(s, np.float32)
        l = np.asarray(l, np.int32)
        order = np.lexsort((-s, l))
        k = len(s)
        ob[i, :k], os_[i, :k], ol[i, :k], cnt[i] = np.asarray(b, np.float32).reshape(-1, 4)[order], s[order], l[order], k
        v = len(gl_i)
        gb[i, :v], gl[i, :v], gc[i] = np.asarray(g, np.float64).reshape(-1, 4), gl_i, v
    return ob, os_, ol, cnt, gb, gl, gc


def _random_images(rng, n, num_classes, k_max, v_max=12, score_levels=64, bad_labels=False):
    """Seeded detections around the ground truth: about half are jittered copies of a gt box (IoUs from ~0.3 to 1,
    many near 0.5), some with the wrong class; scores are multiples of 1/score_levels so ties occur."""
    dets, gts = [], []
    for _ in range(n):
        v = int(rng.integers(0, v_max + 1))
        g0 = rng.uniform(0, 400, (v, 2))
        gwh = rng.uniform(8, 120, (v, 2))
        g = np.concatenate([g0, g0 + gwh], 1)
        gl = rng.integers(0, num_classes, v)
        if bad_labels and v:
            gl[rng.random(v) < 0.2] = rng.choice([-1, num_classes])
        k = int(rng.integers(0, k_max + 1))
        b = np.empty((k, 4))
        lab = rng.integers(0, num_classes, k)
        near = (rng.random(k) < 0.6) & (v > 0)
        src = rng.integers(0, max(v, 1), k)
        for j in range(k):
            if near[j]:
                x0, y0, x1, y1 = g[src[j]]
                w, h = x1 - x0, y1 - y0
                d = rng.uniform(-0.35, 0.35, 4) * [w, h, w, h]
                b[j] = (x0 + d[0], y0 + d[1], x1 + d[2], y1 + d[3])
                if rng.random() < 0.85 and 0 <= gl[src[j]] < num_classes:
                    lab[j] = gl[src[j]]
            else:
                c = rng.uniform(0, 400, 2)
                s = rng.uniform(8, 120, 2)
                b[j] = (c[0], c[1], c[0] + s[0], c[1] + s[1])
        sc = (rng.integers(1, score_levels + 1, k) / score_levels).astype(np.float32)
        dets.append((b, sc, lab))
        gts.append((g, gl))
    return dets, gts


def _batches(dets, gts, num_classes, sizes):
    out, i = [], 0
    vmax = max(1, max(len(g[1]) for g in gts))
    for s in sizes:
        if s:
            out.append(_layout(dets[i:i + s], gts[i:i + s], num_classes, vmax=vmax))
        i += s
    return out


def test_goldens_match_reference():
    """tests/synth.gen_eval_case -> the device batched NMS -> VOCEvaluator equals the rows the reference's voc_eval wrote."""
    import torch
    from tests.synth import gen_eval_case
    from yolov3_tensorflow_b200.utils.eval_utils import VOCEvaluator, pack_gt_rec
    from yolov3_tensorflow_b200.utils.nms_utils import batched_nms_raw
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "eval.npz"))
    for tag in ("a", "b"):
        seed, n, w, h, cn = (int(v) for v in g[f"ev_{tag}_cfg"])
        y_pred, _, gts = gen_eval_case(seed, n, w, h, cn)
        boxes = torch.from_numpy(y_pred[0]).cuda()
        scores = (torch.from_numpy(y_pred[1]) * torch.from_numpy(y_pred[2])).cuda()
        ob, os_, ol, _, cnt = batched_nms_raw(boxes, scores, cn, 20, 0.3, 0.45)
        gt_dict = {100 + i: [[float(v) for v in b[:4]] + [int(l)] for b, l in zip(*gts[i])] for i in range(n)}
        ev = VOCEvaluator(cn)
        ev.add_batch(ob, os_, ol, cnt, *pack_gt_rec(gt_dict, [100 + i for i in range(n)]))
        res = {False: ev.result(False), True: ev.result(True)}
        rows = g[f"voc_{tag}"]
        assert any(r[2] == 0 for r in rows) and len(rows) == 2 * cn        # npos = 0 rows included
        for row in rows:
            c, m07 = int(row[0]), bool(row[1])
            assert_voc_equal([res[m07][c]], [tuple(row[2:])], use_07_metric=m07)


def test_large_random_set_matches_stable_oracle():
    rng = np.random.default_rng(11)
    dets, gts = _random_images(rng, 520, 80, 800)
    assert sum(len(d[1]) for d in dets) >= 200_000
    batches = _batches(dets, gts, 80, [64] * 8 + [8])
    _check(batches, 80)


def _box(x0, y0, x1, y1):
    return [float(x0), float(y0), float(x1), float(y1)]


def test_edge_cases():
    C = 20
    A, B = _box(0, 0, 9, 9), _box(2, 0, 11, 9)
    dets, gts = [], []
    # image 0: class 0: two gt boxes (IoU 0.667); the 2nd detection's best gt is already used -> FP, no fallback to B.
    #          class 2: IoU exactly 0.5 (strict '>': FP), then 0.526 (TP).  class 3: gt, never detected.
    #          class 4: detections without any gt of the class (npos = 0).  class 5: two equal-score hits on one gt.
    #          gt labels -1 and C sit on a class-0 detection and belong to no class.
    db = [A, A, B, _box(0, 0, 9, 19), _box(0, 0, 9, 18), _box(5, 5, 30, 30), _box(40, 40, 60, 60), _box(40, 40, 60, 60)]
    ds = [0.9, 0.8, 0.7, 0.6, 0.5, 0.4, 0.3, 0.3]
    dl = [0, 0, 0, 2, 2, 4, 5, 5]
    gb = [A, B, _box(0, 0, 9, 9), _box(50, 50, 60, 60), _box(40, 40, 60, 60), A, A]
    gl = [0, 0, 2, 3, 5, -1, C]
    dets.append((np.asarray(db), np.asarray(ds, np.float32), np.asarray(dl)))
    gts.append((np.asarray(gb), np.asarray(gl)))
    dets.append((np.zeros((0, 4)), np.zeros(0, np.float32), np.zeros(0, int)))          # image 1: no detections
    gts.append((np.asarray([A]), np.asarray([0])))
    dets.append((np.asarray([A, B]), np.asarray([0.95, 0.2], np.float32), np.asarray([0, 0])))   # image 2: no gt
    gts.append((np.zeros((0, 4)), np.zeros(0, int)))
    # image 3: vmax = 1024 gt boxes, a 400-detection segment of class 6 over them
    rng = np.random.default_rng(3)
    xy = rng.uniform(0, 400, (1024, 2))
    g3 = np.concatenate([xy, xy + rng.uniform(8, 60, (1024, 2))], 1)
    l3 = rng.integers(6, C, 1024)                                       # classes 0-5 stay as image 0 set them
    l3[:300] = 6
    src = rng.integers(0, 300, 400)
    b3 = g3[src] + rng.uniform(-4, 4, (400, 4))
    dets.append((b3, (rng.integers(1, 17, 400) / 16).astype(np.float32), np.full(400, 6)))
    gts.append((g3, l3))
    batch = _layout(dets, gts, C, vmax=1024)
    area, _ = _check([batch], C)
    assert area[2][:2] == (1, 2) and area[2][3] == 0.5                 # class 2: the 0.5 detection is the FP
    assert area[0][:2] == (3, 5) and area[0][2] == 2 / 3               # class 0: A, B found; 2nd A hit and image 2 FPs
    assert area[3] == (1e-6, 1e-6, 0, 0, 0) and area[4][0] == 0 and np.isnan(area[4][2])
    assert area[5][:2] == (1, 2) and area[5][3] == 0.5 and area[6][1] == 400
    # C = 1, with gt labels outside [0, 1)
    dets, gts = _random_images(np.random.default_rng(4), 40, 1, 60, bad_labels=True)
    _check(_batches(dets, gts, 1, [40]), 1)


def test_split_invariance():
    rng = np.random.default_rng(21)
    dets, gts = _random_images(rng, 90, 20, 120)
    for i in (5, 6, 40):
        dets[i] = (np.zeros((0, 4)), np.zeros(0, np.float32), np.zeros(0, int))
    one = _evaluate(_batches(dets, gts, 20, [90]), 20)
    sizes = [1, 4, 2, 33, 17, 33]
    many = _batches(dets, gts, 20, sizes)
    empty = _layout([dets[5]], [gts[5]], 20)
    empty = tuple(a[:0] for a in empty)                                 # a batch of zero images
    split = _evaluate(many[:2] + [empty] + many[2:], 20)
    for a, b in zip(one, split):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            assert np.array_equal(np.asarray(x, np.float64), np.asarray(y, np.float64), equal_nan=True)


def _constructed(rng, counts, num_classes, scores, tp_prob=0.25, extra_gt=8):
    """Detections in the NMS layout whose TP flags are known: a TP sits exactly on its own gt box (boxes 20 px apart,
    so no other gt overlaps it), an FP sits far from every gt, extra unmatched gt boxes sit elsewhere.
    -> (batch arrays, labels, scores, flags in insertion order, npos per class)."""
    n, cap = len(counts), max(1, max(counts))
    ob = np.zeros((n, cap, 4), np.float32); os_ = np.zeros((n, cap), np.float32); ol = np.zeros((n, cap), np.int32)
    lab_all, sc_all, fl_all = [], [], []
    gts = []
    for i, k in enumerate(counts):
        lab = rng.integers(0, num_classes, k)
        sc = scores(k)
        order = np.lexsort((-sc, lab))
        lab, sc = lab[order], sc[order]
        tp = rng.random(k) < tp_prob
        tp[np.cumsum(tp) > 1024 - extra_gt] = False
        b = np.tile(np.asarray([1e5, 1e5, 1e5 + 9, 1e5 + 9], np.float32), (k, 1))
        t = np.flatnonzero(tp)
        cell = np.arange(len(t))
        b[t] = np.stack([(cell % 64) * 20, (cell // 64) * 20, (cell % 64) * 20 + 9, (cell // 64) * 20 + 9], 1)
        ob[i, :k], os_[i, :k], ol[i, :k] = b, sc, lab
        e = np.arange(extra_gt)
        ge = np.stack([e * 20, np.full(extra_gt, 5e4), e * 20 + 9, np.full(extra_gt, 5e4 + 9)], 1)
        gts.append((np.concatenate([b[t].astype(np.float64), ge]), np.concatenate([lab[t], rng.integers(0, num_classes, extra_gt)])))
        lab_all.append(lab); sc_all.append(sc); fl_all.append(tp)
    vmax = max(1, max(len(g[1]) for g in gts))
    gb = np.zeros((n, vmax, 4)); gl = np.full((n, vmax), -1, np.int32); gc = np.zeros(n, np.int32)
    npos = np.zeros(num_classes, np.int64)
    for i, (g, l) in enumerate(gts):
        gb[i, :len(l)], gl[i, :len(l)], gc[i] = g, l, len(l)
        np.add.at(npos, l, 1)
    batch = (ob, os_, ol, np.asarray(counts, np.int32), gb, gl, gc)
    return batch, np.concatenate(lab_all), np.concatenate(sc_all), np.concatenate(fl_all), npos


@pytest.mark.parametrize("case", ["equal", "two", "size1", "tile-1", "tile", "tile+1", "millions"])
def test_sort_stress(case):
    rng = np.random.default_rng(["equal", "two", "size1", "tile-1", "tile", "tile+1", "millions"].index(case))
    quant = lambda k: (rng.integers(1, 65, k) / 64).astype(np.float32)
    C, tile = 20, 4096
    counts, scores, chunks = {
        "equal": ([3000, 2500, 3000], lambda k: np.full(k, 0.5, np.float32), 1),
        "two": ([3000, 2500, 3000], lambda k: np.where(rng.random(k) < 0.5, 0.25, 0.75).astype(np.float32), 1),
        "size1": ([1], quant, 1),
        "tile-1": ([2000, 2095], quant, 1),
        "tile": ([2000, 2096], quant, 1),
        "tile+1": ([2000, 2097], quant, 1),
        "millions": ([1000] * 3000, quant, 6),
    }[case]
    if case == "millions":
        C = 80
    batch, lab, sc, fl, npos = _constructed(rng, counts, C, scores)
    assert case != "size1" or len(lab) == 1
    assert not case.startswith("tile") or len(lab) - tile == {"tile-1": -1, "tile": 0, "tile+1": 1}[case]
    from yolov3_tensorflow_b200.utils.eval_utils import VOCEvaluator
    ev = VOCEvaluator(C)
    n = len(counts)
    step = -(-n // chunks)
    for i in range(0, n, step):
        ev.add_batch(*_cuda(*(a[i:i + step] for a in batch)))
    assert len(ev) == len(lab)
    for m07 in (False, True):
        assert_voc_equal(ev.result(m07), voc_from_flags(lab, sc, fl, npos, C, m07), use_07_metric=m07)


@pytest.mark.parametrize("fp8", [False, True])
def test_end_to_end_detect_raw(fp8):
    """detect_raw at the reference's evaluation settings (400 per class, score 0.01, NMS 0.45) on 16 images at 416^2
    with cfg-2 weights: the device evaluator equals get_preds_gpu's rows + the stable voc_eval."""
    import torch
    import bench
    import yolov3_tensorflow_b200 as pkg
    from oracle import yolov3_oracle as O
    from tests.synth import gen_inputs
    from yolov3_tensorflow_b200.utils.eval_utils import VOCEvaluator, pack_gt_rec
    m = pkg.yolov3(80, O.COCO_ANCHORS, dtype="fp16")
    m.set_params(bench.make_bench_params(specs=m.conv_table(80)), "HWIO")
    if fp8:
        m = m.quantize_fp8(torch.from_numpy(gen_inputs(1000, 4, 416, 416)).cuda())
    x = torch.from_numpy(gen_inputs(5, 16, 416, 416)).cuda()
    rng = np.random.default_rng(6)
    gt_dict = {}
    for i in range(16):
        b, l = O.synth_gt(rng, 416, 416, 80, 30)
        gt_dict[i] = [[float(v) for v in bb[:4]] + [int(ll)] for bb, ll in zip(b, l)]
    ev = VOCEvaluator(80)
    rows = []
    for s in (0, 8):
        _, ob, os_, ol, _, cnt = m.detect_raw(x[s:s + 8], max_boxes=400, score_thresh=0.01, nms_thresh=0.45)
        ev.add_batch(ob, os_, ol, cnt, *pack_gt_rec(gt_dict, list(range(s, s + 8))))
        rows += rows_from_nms(list(range(s, s + 8)), ob.cpu().numpy(), os_.cpu().numpy(), ol.cpu().numpy(), cnt.cpu().numpy())
    assert len(rows) == len(ev) > 1000
    want = voc_eval_stable_all(gt_dict, rows, 80)
    for m07 in (False, True):
        assert_voc_equal(ev.result(m07), want[m07], use_07_metric=m07)
    # eval.py:125-137: AverageMeter over the classes (a class with detections but npos = 0 makes it nan, as there)
    s, n = [0., 0., 0.], [0., 0., 0.]
    for npos, nd, rec, prec, ap in want[0]:
        for k, (v, w) in enumerate(((ap, 1), (rec, npos), (prec, nd))):
            s[k] += v * w
            n[k] += w
    expected = [a / float(b) for a, b in zip(s, n)]
    assert np.allclose(ev.summary(), expected, rtol=0, atol=1e-12, equal_nan=True)
