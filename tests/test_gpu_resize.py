"""GPU tests of the batched evaluation input path (yb_resize_batch, yb_resize_boxes, yb_restore_boxes): bit-exact
against the reference-generated goldens (tests/golden/make_golden_resize.py) and the numpy restatement
(tests/resize_ref.py), which tests/test_resize_host.py pins to the goldens and to cv2."""
import os

import numpy as np
import pytest
import torch

from oracle import yolov3_oracle as O
from tests import resize_ref as R

pytestmark = pytest.mark.gpu


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "resize.npz"))


def _expected_params(img, nw, nh, letterbox):
    h, w = img.shape[:2]
    if letterbox:
        ratio, _, _, dw, dh = R.letterbox_geometry(h, w, nw, nh)
        return [ratio, float(dw), float(dh), 1.0]
    return [w / float(nw), h / float(nh), 0.0, 0.0]


def test_golden_images_bit_exact(golden_dir):
    from yolov3_tensorflow_b200.utils import data_aug as A
    g = _golden(golden_dir)
    for i, (sh, sw, nw, nh) in enumerate(g["cases"].tolist()):
        src = g[f"src{i}"]
        for interp in (0, 1):
            for lb, key in ((True, f"lb{interp}_{i}"), (False, f"st{interp}_{i}")):
                x, p = A.preprocess_batch([src], nw, nh, letterbox=lb, interp=interp)
                assert tuple(x.shape) == (1, nh, nw, 3)
                assert np.array_equal(x[0].cpu().numpy(), R.normalize(g[key])), (i, interp, lb)
                assert p[0].cpu().tolist() == _expected_params(src, nw, nh, lb), (i, interp, lb)
        _, p = A.preprocess_batch([src], nw, nh, letterbox=True)
        assert p[0, :3].cpu().tolist() == g[f"lb_meta{i}"].tolist()
    # test_single_image.py:43-46, the float network input itself
    x, _ = A.preprocess_batch([g["src4"]], *g["cases"][4][2:].tolist(), letterbox=False, interp=1)
    assert np.array_equal(x.cpu().numpy(), g["x_st4"])


def test_golden_box_transforms_bit_exact(golden_dir):
    from yolov3_tensorflow_b200.utils import data_aug as A
    g = _golden(golden_dir)
    for i, (sh, sw, nw, nh) in enumerate(g["cases"].tolist()):
        src, gt = g[f"src{i}"], g[f"gt{i}"]
        for lb, bkey, ikey in ((True, "gt_lb", "lb1_"), (False, "gt_st", "st1_")):
            x, b = A.resize_with_bbox(src, gt, nw, nh, interp=1, letterbox=lb)
            assert np.array_equal(x.cpu().numpy(), R.normalize(g[f"{ikey}{i}"])), (i, lb)
            assert np.array_equal(b.cpu().numpy(), g[f"{bkey}{i}"]), (i, lb)      # incl. the untouched weight column
        # detections back to the source image: 6 valid slots, 2 past the count that must stay as they are
        for lb, key in ((True, "det_lb"), (False, "det_st")):
            _, p = A.preprocess_batch([src], nw, nh, letterbox=lb)
            det = np.concatenate([g[f"det{i}"], np.full((2, 4), -7.5, np.float32)])[None]
            ob = torch.from_numpy(det).cuda()
            cnt = torch.tensor([6], dtype=torch.int32, device="cuda")
            got = A.restore_boxes(ob, cnt, p).cpu().numpy()[0]
            assert np.array_equal(got[:6], g[f"{key}{i}"]), (i, lb)
            assert np.array_equal(got[6:], det[0, 6:]) and np.array_equal(ob.cpu().numpy(), det)


def _mixed_images(golden_dir):
    g = _golden(golden_dir)
    rng = np.random.default_rng(11)
    imgs = [g[f"src{i}"] for i in range(len(g["cases"]))]
    imgs += [rng.integers(0, 256, s, dtype=np.uint8) for s in ((375, 500, 3), (500, 375, 3), (1, 1, 3), (480, 640, 3),
                                                                (416, 416, 3), (208, 832, 3))]
    return imgs


@pytest.mark.parametrize("nw,nh", [(416, 416), (64, 48), (96, 160)])
@pytest.mark.parametrize("letterbox", [True, False])
@pytest.mark.parametrize("interp", [0, 1])
def test_mixed_batch_equals_one_at_a_time_and_oracle(golden_dir, nw, nh, letterbox, interp):
    from yolov3_tensorflow_b200.utils import data_aug as A
    imgs = _mixed_images(golden_dir)
    x, p = A.preprocess_batch(imgs, nw, nh, letterbox=letterbox, interp=interp)
    xs, ps = x.cpu().numpy(), p.cpu().numpy()
    for i, img in enumerate(imgs):
        x1, p1 = A.preprocess_batch([img], nw, nh, letterbox=letterbox, interp=interp)
        assert np.array_equal(xs[i], x1[0].cpu().numpy()) and np.array_equal(ps[i], p1[0].cpu().numpy()), i
        rx, rp = R.preprocess(img, nw, nh, letterbox, interp)
        assert np.array_equal(xs[i], rx), i
        assert ps[i].tolist() == _expected_params(img, nw, nh, letterbox) and tuple(ps[i, :3]) == rp
    # out=: the same bytes written into a caller's buffer
    out = torch.full((len(imgs), nh, nw, 3), float("nan"), device="cuda")
    x2, _ = A.preprocess_batch(imgs, nw, nh, letterbox=letterbox, interp=interp, out=out)
    assert x2.data_ptr() == out.data_ptr() and np.array_equal(out.cpu().numpy(), xs)


@pytest.mark.parametrize("sh,sw,nw,nh", [(480, 640, 416, 416), (1080, 1920, 608, 608), (333, 500, 416, 416),
                                         (500, 333, 416, 416), (75, 100, 128, 96), (1, 1, 64, 32)])
def test_nearest_letterbox_equals_letterbox_preprocess(sh, sw, nw, nh):
    from yolov3_tensorflow_b200.utils import data_aug as A
    img = np.random.default_rng(sh * sw).integers(0, 256, (sh, sw, 3), dtype=np.uint8)
    x1, ratio, dw, dh = A.letterbox_preprocess(img, nw, nh)
    x, p = A.preprocess_batch([img, img[: sh // 2 + 1]], nw, nh, letterbox=True, interp=0)
    assert np.array_equal(x[0].cpu().numpy(), x1[0].cpu().numpy())
    assert p[0].cpu().tolist() == [ratio, float(dw), float(dh), 1.0]


def _model():
    import bench
    import yolov3_tensorflow_b200 as pkg
    m = pkg.yolov3(80, O.COCO_ANCHORS, dtype="fp16")
    m.set_params(bench.make_bench_params(specs=m.conv_table(80)), "HWIO")
    return m


def _voc_like_images(seed, n):
    """uint8 BGR sources of VOC's two common shapes, smooth enough for the bench weights to fire."""
    from tests.synth import gen_inputs
    imgs = []
    for i in range(n):
        h, w = (375, 500) if i % 2 == 0 else (500, 375)
        imgs.append(np.ascontiguousarray((gen_inputs(seed + i, 1, h, w)[0] * 255).astype(np.uint8)))
    return imgs


@pytest.mark.parametrize("letterbox", [True, False])
def test_restore_boxes_on_detect_raw(letterbox):
    from yolov3_tensorflow_b200.utils import data_aug as A
    m = _model()
    imgs = _voc_like_images(30, 4)
    x, p = A.preprocess_batch(imgs, 416, 416, letterbox=letterbox, interp=1)
    _, ob, _, _, _, cnt = m.detect_raw(x, max_boxes=50, score_thresh=0.01, nms_thresh=0.45)
    before = ob.cpu().numpy()
    got = A.restore_boxes(ob, cnt, p).cpu().numpy()
    counts = cnt.cpu().numpy()
    assert counts.sum() > 0
    for i, img in enumerate(imgs):
        k = int(counts[i])
        row = tuple(p[i, :3].cpu().tolist())
        assert np.array_equal(got[i, :k], R.restore_boxes(before[i, :k], row, letterbox)), i
        assert np.array_equal(got[i, k:], before[i, k:])
    assert np.array_equal(ob.cpu().numpy(), before)                   # not in place by default
    A.restore_boxes(ob, cnt, p, inplace=True)
    assert np.array_equal(ob.cpu().numpy(), got)


@pytest.mark.parametrize("letterbox", [True, False])
def test_val_batch_matches_process_box_on_golden_boxes(golden_dir, letterbox):
    """The golden cases 5 and 7 target 64 x 32: val_batch's images equal the restatement, and its y_true equal
    process_box on the reference's own resize_with_bbox boxes (with mix-up weights and an image without boxes)."""
    from yolov3_tensorflow_b200.utils import data_utils as D
    g = _golden(golden_dir)
    W, H, C = 64, 32, 20
    idx = [5, 7, 5, 7]
    assert all(tuple(g["cases"][i][2:]) == (W, H) for i in idx)
    imgs = [g[f"src{i}"] for i in idx]
    rng = np.random.default_rng(5)
    key = "gt_lb" if letterbox else "gt_st"
    weights = [np.ones(4, np.float32), np.ones(4, np.float32), rng.uniform(0.5, 1, 4).astype(np.float32), None]
    boxes = [g[f"gt{i}"][:, :4] for i in idx]                         # parse_line's [V, 4]: the weight 1 is added
    boxes[2] = np.concatenate([boxes[2], weights[2][:, None]], 1)     # mix-up weights are carried
    boxes[3] = boxes[3][:0]                                            # an image without ground truth
    labels = [rng.integers(0, C, len(b)) for b in boxes]
    x, y13, y26, y52 = D.val_batch(imgs, boxes, labels, [W, H], C, O.COCO_ANCHORS, letterbox_resize=letterbox)
    for k, (i, l) in enumerate(zip(idx, labels)):
        rx, _ = R.preprocess(imgs[k], W, H, letterbox, 1)
        assert np.array_equal(x[k].cpu().numpy(), rx), k
        tb = g[f"{key}{i}"][: len(l)].copy()
        if weights[k] is not None:
            tb[:, 4] = weights[k]
        ref = O.process_box(tb, l, [W, H], C, O.COCO_ANCHORS)
        for y, r in zip((y13, y26, y52), ref):
            assert np.array_equal(y[k].cpu().numpy(), r), k


def test_bad_arguments_raise_value_error():
    from yolov3_tensorflow_b200.utils import data_aug as A
    from yolov3_tensorflow_b200.utils import data_utils as D
    ok = np.zeros((10, 20, 3), np.uint8)
    with pytest.raises(ValueError):
        A.preprocess_batch([ok, np.zeros((0, 20, 3), np.uint8)], 32, 32)             # zero-sized image
    with pytest.raises(ValueError):
        A.preprocess_batch([np.zeros((1, 3000, 3), np.uint8)], 32, 32, letterbox=True)   # letterboxes to 0 rows
    with pytest.raises(ValueError):
        A.preprocess_batch([ok], 32, 32, interp=2)
    with pytest.raises(ValueError):
        A.preprocess_batch([ok.astype(np.float32)], 32, 32)
    with pytest.raises(ValueError):
        A.preprocess_batch([ok[..., :2]], 32, 32)
    with pytest.raises(ValueError):
        A.preprocess_batch([], 32, 32)
    with pytest.raises(ValueError):
        A.preprocess_batch([ok], 0, 32)
    with pytest.raises(ValueError):
        A.preprocess_batch([ok], 32, 32, out=torch.empty((1, 32, 31, 3), device="cuda"))
    with pytest.raises(ValueError):
        A.resize_with_bbox(ok, np.zeros((2, 3), np.float32), 32, 32)
    with pytest.raises(ValueError):
        A.restore_boxes(torch.zeros((1, 4, 4), device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda"),
                        torch.zeros((1, 4), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        D.val_batch([ok], [np.zeros((1, 4), np.float32)], [np.zeros(1, np.int64)], [100, 96], 20, O.COCO_ANCHORS)
    # stretch of the sliver that cannot be letterboxed is fine
    x, _ = A.preprocess_batch([np.zeros((1, 3000, 3), np.uint8)], 32, 32, letterbox=False)
    assert np.array_equal(x.cpu().numpy(), np.zeros((1, 32, 32, 3), np.float32))


@pytest.mark.parametrize("letterbox", [True, False])
def test_end_to_end_uint8_to_voc_evaluator_equals_host_path(letterbox):
    """uint8 images -> preprocess_batch -> detect_raw -> VOCEvaluator gives what the host path (cv2 where it imports,
    else the restatement; + float32 upload) gives: the same input bytes, detections and per-class results."""
    from yolov3_tensorflow_b200.utils import data_aug as A
    from yolov3_tensorflow_b200.utils.eval_utils import VOCEvaluator, pack_gt_rec
    try:
        import cv2
    except ImportError:
        cv2 = None
    m = _model()
    imgs = _voc_like_images(50, 8)
    rng = np.random.default_rng(9)
    gt = {}
    for i in range(8):
        b, l = O.synth_gt(rng, 416, 416, 80, 12)
        gt[i] = [[float(v) for v in bb[:4]] + [int(ll)] for bb, ll in zip(b, l)]

    def host(img):
        if cv2 is None:
            return R.preprocess(img, 416, 416, letterbox, 1)[0]
        if letterbox:
            ratio = min(416 / img.shape[1], 416 / img.shape[0])
            rw, rh = int(ratio * img.shape[1]), int(ratio * img.shape[0])
            pad = np.full((416, 416, 3), 128, np.uint8)
            dw, dh = int((416 - rw) / 2), int((416 - rh) / 2)
            pad[dh: rh + dh, dw: rw + dw] = cv2.resize(img, (rw, rh), interpolation=1)
        else:
            pad = cv2.resize(img, (416, 416), interpolation=1)
        return np.asarray(cv2.cvtColor(pad, cv2.COLOR_BGR2RGB), np.float32) / 255.

    results, outs = [], []
    for path in ("device", "host"):
        ev = VOCEvaluator(80)
        xs = []
        for s in (0, 4):
            if path == "device":
                x, _ = A.preprocess_batch(imgs[s:s + 4], 416, 416, letterbox=letterbox, interp=1)
            else:
                x = torch.from_numpy(np.stack([host(im) for im in imgs[s:s + 4]]).astype(np.float32)).cuda()
            xs.append(x.cpu().numpy())
            _, ob, os_, ol, _, cnt = m.detect_raw(x, max_boxes=400, score_thresh=0.01, nms_thresh=0.45)
            outs.append([t.cpu().numpy() for t in (ob, os_, ol, cnt)])
            ev.add_batch(ob, os_, ol, cnt, *pack_gt_rec(gt, list(range(s, s + 4))))
        results.append((np.concatenate(xs), ev.result(False), ev.result(True), len(ev)))
    (xd, r0d, r1d, nd), (xh, r0h, r1h, nh) = results
    assert np.array_equal(xd, xh)
    assert nd == nh > 0
    for (db, ds, dl, dc), (hb, hs, hl, hc) in zip(outs[:2], outs[2:]):
        assert np.array_equal(dc, hc)
        for i, k in enumerate(dc.tolist()):
            assert np.array_equal(db[i, :k], hb[i, :k]) and np.array_equal(ds[i, :k], hs[i, :k])
            assert np.array_equal(dl[i, :k], hl[i, :k])
    for ra, rb in ((r0d, r0h), (r1d, r1h)):
        for a, b in zip(ra, rb):
            for u, v in zip(a, b):
                assert np.array_equal(np.asarray(u, np.float64), np.asarray(v, np.float64), equal_nan=True)
