"""GPU tests of the training augmentation (yb_augment_batch, yb_flip_batch, utils.data_aug.augment_train_batch and
the single-image functions): byte for byte against the reference-generated goldens (tests/golden/make_golden_augment.py)
and the numpy restatement (tests/augment_ref.py) from the same seeds, RNG states included."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import yolov3_oracle as O
from tests import augment_ref as A
from tests import resize_ref as R
from tests.test_augment_host import assert_rng_states, golden_inputs, seed_golden

pytestmark = pytest.mark.gpu


def _images(packed):
    return [packed.image(i).cpu().numpy() for i in range(packed.n)]


def _batch_case(seed, sizes, mix, nbox):
    rng = np.random.default_rng(seed)
    imgs, boxes, labels = [], [], []
    for (h, w), v in zip(sizes, nbox):
        imgs.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        x0, x1 = rng.uniform(0, w, v), rng.uniform(0, w, v)
        y0, y1 = rng.uniform(0, h, v), rng.uniform(0, h, v)
        b = np.stack([np.minimum(x0, x1), np.minimum(y0, y1), np.maximum(x0, x1) + 2, np.maximum(y0, y1) + 2], 1)
        boxes.append(b.astype(np.float32).reshape(-1, 4))
        labels.append(rng.integers(0, 20, v).astype(np.int64))
    return imgs, boxes, labels, mix


def _restate(imgs, boxes, labels, mix):
    recs = []
    for i in range(len(imgs)):
        j = mix[i]
        recs.append(A.train_image(imgs[i], boxes[i], labels[i],
                                  *((imgs[j], boxes[j], labels[j]) if j is not None else ())))
    return recs


def _assert_batch_equals(out, recs):
    packed, bx, lb, interp, flip = out
    for i, (got, rec) in enumerate(zip(_images(packed), recs)):
        assert np.array_equal(got, rec["img"]), i
        assert bx[i].dtype == rec["boxes"].dtype and np.array_equal(bx[i], rec["boxes"]), i
        assert np.array_equal(lb[i], rec["labels"][:len(rec["boxes"])]), i
        assert interp[i] == rec["interp"] and flip[i] == rec["flip"], i


def test_batch_matches_reference_golden(golden_dir):
    from yolov3_tensorflow_b200.utils import data_aug as D
    g = np.load(os.path.join(golden_dir, "augment.npz"))
    imgs, boxes, labels, mix = golden_inputs(g)
    seed_golden()
    packed, bx, lb, interp, flip = D.augment_train_batch(imgs, boxes, labels, mix_with=mix)
    assert_rng_states(g, len(imgs) - 1)
    for i, got in enumerate(_images(packed)):
        assert np.array_equal(got, g[f"crop_img{i}"]), i
        assert bx[i].dtype == g[f"boxes{i}"].dtype and np.array_equal(bx[i], g[f"boxes{i}"]), i
        assert np.array_equal(lb[i], g[f"labels{i}"][:len(bx[i])]), i
        assert interp[i] == int(g[f"interp{i}"]) and flip[i] == bool(g[f"flip{i}"]), i


SIZES = [(1, 1), (7, 33), (375, 500), (64, 31), (1, 1), (500, 375), (33, 65), (17, 129), (96, 95), (3, 200)]
MIX = [None, 5, 3, None, 2, None, 0, 9, None, 7]
NBOX = [0, 3, 5, 2, 0, 4, 0, 1, 6, 2]


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_mixed_batch_matches_restatement(seed):
    """1 x 1 images, odd widths, mix-up pairs of different sizes, box-less images, with and without expand."""
    from yolov3_tensorflow_b200.utils import data_aug as D
    case = _batch_case(seed, SIZES, MIX, NBOX)
    np.random.seed(seed); random.seed(seed + 100)
    recs = _restate(*case)
    ref_np, ref_py = np.random.get_state(), random.getstate()
    assert any(r["expand"] is None for r in recs) and any(r["expand"] is not None for r in recs)
    np.random.seed(seed); random.seed(seed + 100)
    out = D.augment_train_batch(*case[:3], mix_with=case[3])
    st = np.random.get_state()
    assert np.array_equal(st[1], ref_np[1]) and st[2] == ref_np[2] and random.getstate() == ref_py
    _assert_batch_equals(out, recs)


def test_batch_equals_single_image_functions():
    from yolov3_tensorflow_b200.utils import data_aug as D
    imgs, boxes, labels, _ = _batch_case(9, [(120, 90), (75, 100)], None, [3, 2])
    for expand_seed in (0, 1, 2, 3):
        np.random.seed(expand_seed); random.seed(7)
        packed, bx, lb, interp, flip = D.augment_train_batch(imgs, boxes, labels, mix_with=[1, None])
        np.random.seed(expand_seed); random.seed(7)
        img, b = D.mix_up(imgs[0], imgs[1], boxes[0], boxes[1])
        img = D.random_color_distort(img)
        if np.random.uniform(0, 1) > 0.5:
            img, b = D.random_expand(img, b, 4)
        b, (x0, y0, w, h) = D.random_crop_with_constraints(b, (img.shape[1], img.shape[0]))
        assert np.array_equal(img[y0: y0 + h, x0: x0 + w].cpu().numpy(), packed.image(0).cpu().numpy())
        assert np.array_equal(b, bx[0]) and np.random.randint(0, 5) == interp[0]
        rimg = torch.rand((16, 24, 3), device="cuda")
        fimg, fb = D.random_flip(rimg, b.copy(), px=0.5)
        assert torch.equal(fimg, rimg.flip(1) if flip[0] else rimg)
        assert np.array_equal(fb, A.flip_boxes(b, 24, 16, bool(flip[0])))


def test_decoded_batch_goes_in_without_upload(golden_dir):
    from yolov3_tensorflow_b200.utils import data_aug as D
    files = [os.path.join(golden_dir, f) for f in ("dog.jpg", "messi.jpg")]
    packed = D.decode_jpeg_batch(files)
    host = _images(packed)
    boxes = [np.array([[100, 120, 300, 400]], np.float32), np.array([[50, 40, 200, 300], [300, 20, 500, 330]],
                                                                     np.float32)]
    labels = [np.array([16]), np.array([0, 32])]
    np.random.seed(4); random.seed(4)
    out = D.augment_train_batch(packed, boxes, labels, mix_with=[1, None])
    assert out[0].h2d_bytes == 2 * 80                     # only the parameter table crossed
    np.random.seed(4); random.seed(4)
    _assert_batch_equals(out, _restate(host, boxes, labels, [1, None]))


def _all_bgr(width):
    v = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([v & 255, (v >> 8) & 255, v >> 16], -1).astype(np.uint8)
    rows = -(-len(img) // width)
    return np.concatenate([img, np.zeros((rows * width - len(img), 3), np.uint8)]).reshape(rows, width, 3)


@pytest.mark.parametrize("color", [None, (0, 0, 1.0, 1.0), (20, 7, 1.3, 0.7), (-25, -18, 0.6, 1.45), (31, 17, 1.5, 0.5)])
def test_every_bgr_value_through_each_op_combination(color):
    """All 2^24 BGR values, at widths 4096 (the vector path of HSV2BGR only) and 47 (both paths)."""
    from yolov3_tensorflow_b200.utils import data_aug as D
    for width in (4096, 47):
        img = _all_bgr(width)
        packed = D.PackedImages([img])
        h, w = img.shape[:2]
        got = D._augment_launch(packed, [D._augment_param(0, h, w, color=color)]).image(0).cpu().numpy()
        if color is None:
            ref = img
        else:
            b, hue, s, v = color
            ref = A.color_pixels(img, {"bright": b, "hue": hue, "sat": s, "val": v})
        assert np.array_equal(got, ref), (color, width)


@pytest.mark.parametrize("interp", [0, 1])
def test_chain_through_resize_flip_and_process_box(interp):
    """augment_train_batch -> preprocess_batch(interp) -> flip_batch -> process_box_batch equals the host chain."""
    from yolov3_tensorflow_b200.utils import data_aug as D
    from yolov3_tensorflow_b200.utils import data_utils as U
    sizes = [(375, 500), (500, 375), (64, 31), (96, 95), (200, 120), (33, 65)]
    case = _batch_case(11 + interp, sizes, [1, None, None, 0, 5, None], [3, 4, 1, 0, 2, 5])
    S, cn = 96, 20
    np.random.seed(interp); random.seed(interp)
    recs = _restate(*case)
    np.random.seed(interp); random.seed(interp)
    packed, bx, lb, _, flip = D.augment_train_batch(*case[:3], mix_with=case[3])
    x, _ = D.preprocess_batch(packed, S, S, letterbox=True, interp=interp)
    hb, hl, hc = U.pack_gt([b.astype(np.float32) for b in bx], lb)
    b, c = hb.cuda(), hc.cuda()
    from yolov3_tensorflow_b200._lib import lib, check, ptr, stream_handle
    check(lib.yb_resize_boxes(ptr(b), ptr(c), packed.n, int(b.shape[1]), 5, ptr(packed.desc_dev), S, S, 1,
                              stream_handle()), "yb_resize_boxes")
    D.flip_batch(x, flip, b, c)
    ys = U.process_box_batch(b, hl, c, [S, S], cn, O.COCO_ANCHORS)
    ref_boxes = []
    for i, rec in enumerate(recs):
        xr, _ = R.preprocess(rec["img"], S, S, True, interp)
        assert np.array_equal(x[i].cpu().numpy(), A.flip_pixels(xr, rec["flip"])), i
        rb = R.resize_boxes(rec["boxes"].astype(np.float32), *rec["img"].shape[:2], S, S, True)
        rb = A.flip_boxes(rb, np.float32(S), np.float32(S), rec["flip"])
        assert np.array_equal(b[i, :len(rb)].cpu().numpy(), rb), i
        ref_boxes.append(rb)
    rb, rl, rc = U.pack_gt(ref_boxes, [r["labels"][:len(r["boxes"])] for r in recs])
    for y, r in zip(ys, U.process_box_batch(rb, rl, rc, [S, S], cn, O.COCO_ANCHORS)):
        assert torch.equal(y, r)


def test_bad_inputs_raise_value_error():
    from yolov3_tensorflow_b200.utils import data_aug as D
    imgs = [np.zeros((8, 8, 3), np.uint8), np.zeros((4, 6, 3), np.uint8)]
    boxes = [np.array([[1, 1, 5, 5]], np.float32), np.zeros((0, 4), np.float32)]
    labels = [np.array([1]), np.array([], np.int64)]
    with pytest.raises(ValueError):
        D.augment_train_batch(imgs, boxes[:1], labels)
    with pytest.raises(ValueError):
        D.augment_train_batch(imgs, boxes, labels, mix_with=[2, None])
    with pytest.raises(ValueError):
        D.augment_train_batch(imgs, [np.ones((1, 5), np.float32), boxes[1]], labels)
    with pytest.raises(ValueError):
        D.augment_train_batch(imgs, boxes, [np.array([1, 2]), labels[1]])
    with pytest.raises(ValueError):
        D.augment_train_batch([np.zeros((8, 8), np.uint8)], boxes[:1], labels[:1])
    packed = D.PackedImages(imgs)
    with pytest.raises(ValueError):                       # crop window off the canvas, refused by yb_augment_batch
        D._augment_launch(packed, [D._augment_param(0, 8, 8, crop=(1, 0, 8, 8))])
    with pytest.raises(ValueError):
        D._augment_launch(packed, [D._augment_param(0, 8, 8, expand=(8, 8, 1, 0))])
    x = torch.zeros((2, 8, 8, 3), device="cuda")
    with pytest.raises(ValueError):
        D.flip_batch(x.half(), [1, 0])
    with pytest.raises(ValueError):
        D.flip_batch(x, [1, 0, 1])
    with pytest.raises(ValueError):
        D.flip_batch(x, [1, 0], torch.zeros((2, 3, 5), device="cuda"))
