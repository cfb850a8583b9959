"""CPU tests of the training augmentation: the numpy restatement (tests/augment_ref.py) equals OpenCV's two 8-bit HSV
conversions on every value and the reference-generated goldens (tests/golden/make_golden_augment.py) byte for byte,
including both RNG states after every image; yb_augment_batch / yb_flip_batch reject bad arguments before any
device work."""
import ctypes as C
import os
import random

import numpy as np
import pytest

from tests import augment_ref as A
from tests import resize_ref as R


def test_bgr2hsv_equals_cv2_on_every_value():
    cv2 = pytest.importorskip("cv2")
    v = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([v & 255, (v >> 8) & 255, v >> 16], -1).astype(np.uint8).reshape(4096, 4096, 3)
    assert np.array_equal(A.bgr2hsv(img), cv2.cvtColor(img, cv2.COLOR_BGR2HSV))


def _all_hsv():
    h, s, v = np.meshgrid(np.arange(180), np.arange(256), np.arange(256), indexing="ij")
    return np.stack([h, s, v], -1).astype(np.uint8)


def test_hsv2bgr_equals_cv2_on_every_value():
    """Both of OpenCV's code paths: rows of 256 pixels go through the vector code only, rows of 1 pixel through the
    scalar code only."""
    cv2 = pytest.importorskip("cv2")
    hsv = _all_hsv()
    wide = hsv.reshape(180 * 256, 256, 3)
    assert np.array_equal(A.hsv2bgr(wide), cv2.cvtColor(wide, cv2.COLOR_HSV2BGR))
    tall = hsv.reshape(-1, 1, 3)
    assert np.array_equal(A.hsv2bgr(tall), cv2.cvtColor(tall, cv2.COLOR_HSV2BGR))


def test_hsv2bgr_column_rule_matches_cv2_across_widths():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    for w in (1, 31, 32, 33, 63, 64, 65, 100, 375, 500):
        img = rng.integers(0, 256, (7, w, 3), dtype=np.uint8)
        img[..., 0] %= 180
        assert np.array_equal(A.hsv2bgr(img), cv2.cvtColor(img, cv2.COLOR_HSV2BGR)), w


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "augment.npz"))


def golden_inputs(g):
    n = len(g["sizes"])
    imgs = [g[f"src{i}"] for i in range(n)]
    boxes = [g[f"gt{i}"] for i in range(n)]
    labels = [g[f"lab{i}"] for i in range(n)]
    mix = [None if m < 0 else int(m) for m in g["mix"].tolist()]
    return imgs, boxes, labels, mix


def seed_golden():
    np.random.seed(2026)
    random.seed(1234)
    np.random.beta(1.5, 1.5), np.random.uniform(0, 1)        # the golden script's scalar-type check
    np.random.seed(2026)


def assert_rng_states(g, i):
    st = np.random.get_state()
    assert np.array_equal(st[1], g[f"np_keys{i}"]) and st[2] == int(g[f"np_pos{i}"]), i
    assert np.array_equal(np.asarray(random.getstate()[1], np.int64), g[f"py_state{i}"]), i


def test_restatement_matches_reference_golden(golden_dir):
    g = _golden(golden_dir)
    assert str(g["numpy_version"]).startswith("2.")
    imgs, boxes, labels, mix = golden_inputs(g)
    seed_golden()
    for i in range(len(imgs)):
        j = mix[i]
        rec = A.train_image(imgs[i], boxes[i], labels[i], *((imgs[j], boxes[j], labels[j]) if j is not None else ()))
        assert np.array_equal(rec["img"], g[f"crop_img{i}"]), i
        assert rec["boxes"].dtype == g[f"boxes{i}"].dtype and np.array_equal(rec["boxes"], g[f"boxes{i}"]), i
        assert np.array_equal(rec["labels"], g[f"labels{i}"]), i
        assert rec["crop"] == tuple(g[f"crop{i}"].tolist()), i
        assert rec["interp"] == int(g[f"interp{i}"]) and rec["flip"] == bool(g[f"flip{i}"]), i
        assert_rng_states(g, i)
        if rec["interp"] in (0, 1) and rec["img"].size:
            # the host chain after the crop: letterbox resize, then the flip of the resized image
            padded, ratio, dw, dh = R.letterbox_resize(rec["img"], 64, 64, rec["interp"])
            assert np.array_equal(A.flip_pixels(padded, rec["flip"]), g[f"final_img{i}"]), i
            b = rec["boxes"].copy()
            s = b.dtype.type
            b[:, [0, 2]] = b[:, [0, 2]] * s(ratio) + s(dw)
            b[:, [1, 3]] = b[:, [1, 3]] * s(ratio) + s(dh)
            assert np.array_equal(A.flip_boxes(b, s(64), s(64), rec["flip"]), g[f"final_boxes{i}"]), i


def test_golden_covers_the_traps(golden_dir):
    """An empty crop (1 x 1 image), boxes dropped by the crop while their labels stay, float64 boxes after a mix-up,
    images without boxes and without expand."""
    g = _golden(golden_dir)
    n = len(g["sizes"])
    assert any(g[f"crop_img{i}"].size == 0 for i in range(n))
    assert any(len(g[f"labels{i}"]) > len(g[f"boxes{i}"]) for i in range(n))
    assert {g[f"boxes{i}"].dtype for i in range(n)} == {np.dtype(np.float32), np.dtype(np.float64)}
    assert any(int(s[2]) == 0 for s in g["sizes"])
    assert {int(g[f"interp{i}"]) for i in range(n)} >= {0, 1}


def test_crop_raises_like_the_reference_at_full_size(monkeypatch):
    """random.randrange(0) when a trial window is as tall as the image: the reference raises, so does this."""
    from yolov3_tensorflow_b200.utils import data_aug
    monkeypatch.setattr(random, "uniform", lambda a, b: 1.0)
    with pytest.raises(ValueError):
        data_aug.random_crop_with_constraints(np.zeros((0, 5), np.float32), (40, 30))


@pytest.fixture(scope="module")
def lib():
    from yolov3_tensorflow_b200 import _lib
    return _lib


def _param(lib, **kw):
    p = lib.AugmentParam()
    base = dict(out_h=10, out_w=20, canvas_h=10, canvas_w=20, src1=0, src2=-1, w1=1.0, saturation=1.0, value=1.0)
    for k, v in {**base, **kw}.items():
        setattr(p, k, v)
    return p


def _augment_rc(lib, params, desc=((0, 10, 20, 60),), nbytes=1 << 20, out_bytes=1 << 20, fake_params=None,
                out_desc=None):
    desc = np.ascontiguousarray(desc, np.int64)
    table = (lib.AugmentParam * len(params))(*params)
    fake = C.c_void_p(1 << 20)                      # never dereferenced: validation precedes any device work
    return lib.lib.yb_augment_batch(fake, nbytes, desc.ctypes.data_as(C.c_void_p), fake, len(desc),
                                    C.cast(table, C.c_void_p), fake if fake_params is None else fake_params,
                                    len(params), fake, out_bytes, fake if out_desc is None else out_desc, None)


def test_augment_batch_rejects_bad_arguments(lib):
    P = lambda **kw: _param(lib, **kw)                # noqa: E731
    assert _augment_rc(lib, [P()], desc=[(0, 0, 20, 60)]) == -1                  # zero-sized image
    assert _augment_rc(lib, [P()], desc=[(0, 10, 20, 59)]) == -1                 # pitch < 3 * w
    assert _augment_rc(lib, [P()], desc=[(64, 10, 20, 60)], nbytes=600) == -1    # past the end of the buffer
    assert _augment_rc(lib, [P(src1=1)]) == -1                                   # no such image
    assert _augment_rc(lib, [P(src2=1)]) == -1
    assert _augment_rc(lib, [P(src2=-2)]) == -1
    assert b"reads images" in lib.lib.yb_last_error_string()
    assert _augment_rc(lib, [P(canvas_h=9)]) == -1                               # canvas smaller than the image
    assert _augment_rc(lib, [P(canvas_h=20, off_y=11, out_h=10)]) == -1          # expand offset off the canvas
    assert _augment_rc(lib, [P(canvas_h=20, off_x=-1)]) == -1
    assert b"expand offset" in lib.lib.yb_last_error_string()
    assert _augment_rc(lib, [P(crop_x=1)]) == -1                                 # crop window off the canvas
    assert _augment_rc(lib, [P(crop_y=-1, out_h=5)]) == -1
    assert _augment_rc(lib, [P(out_h=11)]) == -1
    assert b"crop" in lib.lib.yb_last_error_string()
    assert _augment_rc(lib, [P()], out_bytes=599) == -1                          # output past its buffer
    assert _augment_rc(lib, [P(out_offset=-16)]) == -1
    assert _augment_rc(lib, [P(color=2)]) == -1
    assert _augment_rc(lib, [P(fill=256)]) == -1
    assert _augment_rc(lib, [P(saturation=float("nan"))]) == -1
    assert _augment_rc(lib, [P()], fake_params=C.c_void_p((1 << 20) + 4)) == -1  # parameter table not 8-byte aligned
    assert _augment_rc(lib, [P()], out_desc=C.c_void_p((1 << 20) + 4)) == -1
    assert _augment_rc(lib, []) == -1


def test_flip_batch_rejects_bad_arguments(lib):
    fake = C.c_void_p(1 << 20)
    f = lib.lib.yb_flip_batch
    assert f(fake, 0, 8, 8, 4, fake, None, None, 0, 0, None) == -1               # no images
    assert f(fake, 1, 0, 8, 4, fake, None, None, 0, 0, None) == -1
    assert f(fake, 1, 8, 8, 2, fake, None, None, 0, 0, None) == -1               # neither uint8 nor float32
    assert f(C.c_void_p((1 << 20) + 2), 1, 8, 8, 4, fake, None, None, 0, 0, None) == -1
    assert f(fake, 1, 8, 8, 4, None, None, None, 0, 0, None) == -1               # no flags
    assert f(fake, 1, 8, 8, 4, fake, fake, None, 4, 5, None) == -1               # boxes without counts
    assert f(fake, 1, 8, 8, 4, fake, fake, fake, 4, 3, None) == -1               # box_ld < 4
