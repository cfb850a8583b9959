"""CPU tests of the batched evaluation input path: the numpy restatement (tests/resize_ref.py) equals the
reference-generated goldens (tests/golden/make_golden_resize.py) bit for bit and live cv2.resize over random shapes;
yb_resize_batch / yb_resize_boxes / yb_restore_boxes reject bad arguments before any device work."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import resize_ref as R


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "resize.npz"))


def test_restatement_matches_reference_golden_images(golden_dir):
    g = _golden(golden_dir)
    for i, (sh, sw, nw, nh) in enumerate(g["cases"].tolist()):
        src = g[f"src{i}"]
        assert src.shape == (sh, sw, 3)
        for interp in (0, 1):
            padded, ratio, dw, dh = R.letterbox_resize(src, nw, nh, interp)
            assert np.array_equal(padded, g[f"lb{interp}_{i}"]), (i, interp)
            assert (ratio, dw, dh) == tuple(g[f"lb_meta{i}"].tolist())
            assert np.array_equal(R.cv2_resize(src, nw, nh, interp), g[f"st{interp}_{i}"]), (i, interp)
    x, params = R.preprocess(g["src4"], *g["cases"][4][2:].tolist(), letterbox=False, interp=1)
    assert np.array_equal(x[None], g["x_st4"])
    assert params[:2] == (61 / 48.0, 33 / 40.0)


def test_restatement_matches_reference_golden_boxes(golden_dir):
    g = _golden(golden_dir)
    for i, (sh, sw, nw, nh) in enumerate(g["cases"].tolist()):
        gt = g[f"gt{i}"]
        for lb, key in ((True, "gt_lb"), (False, "gt_st")):
            got = R.resize_boxes(gt, sh, sw, nw, nh, lb)
            assert got.dtype == np.float32 and np.array_equal(got, g[f"{key}{i}"]), (i, lb)
        _, lp = R.preprocess(g[f"src{i}"], nw, nh, True, 1)
        _, sp = R.preprocess(g[f"src{i}"], nw, nh, False, 1)
        assert np.array_equal(R.restore_boxes(g[f"det{i}"], lp, True), g[f"det_lb{i}"]), i
        assert np.array_equal(R.restore_boxes(g[f"det{i}"], sp, False), g[f"det_st{i}"]), i


def test_restatement_matches_live_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    shapes = [(1, 1, 5, 3), (2, 2, 1, 1), (375, 500, 416, 416), (500, 375, 416, 416), (1080, 1920, 608, 608),
              (832, 832, 416, 416), (3, 1, 1, 40)]
    shapes += [tuple(int(v) for v in rng.integers(1, 260, 4)) for _ in range(60)]
    for sh, sw, nw, nh in shapes:
        img = rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8)
        for interp in (0, 1):
            assert np.array_equal(R.cv2_resize(img, nw, nh, interp),
                                  cv2.resize(img, (nw, nh), interpolation=interp)), (sh, sw, nw, nh, interp)


@pytest.fixture(scope="module")
def lib():
    from yolov3_tensorflow_b200 import _lib
    return _lib


def _resize_rc(lib, desc, n=None, new_h=32, new_w=32, letterbox=1, interp=1, nbytes=1 << 20, params=None):
    desc = np.ascontiguousarray(desc, np.int64)
    fake = C.c_void_p(1 << 20)                      # never dereferenced: validation precedes any device work
    return lib.lib.yb_resize_batch(fake, nbytes, desc.ctypes.data_as(C.c_void_p), fake,
                                   len(desc) if n is None else n, new_h, new_w, letterbox, interp, fake, params, None)


def test_resize_batch_rejects_bad_arguments(lib):
    ok = [[0, 10, 20, 60]]
    assert _resize_rc(lib, [[0, 0, 20, 60]]) == -1                        # zero-sized image
    assert _resize_rc(lib, [[0, 10, 0, 0]]) == -1
    assert _resize_rc(lib, [[0, 1, 1000, 3000]], letterbox=1) == -1       # int() truncation leaves a 0-row resize
    assert b"empty" in lib.lib.yb_last_error_string()
    assert _resize_rc(lib, ok, interp=2) == -1
    assert _resize_rc(lib, ok, letterbox=2) == -1
    assert _resize_rc(lib, ok, new_h=0) == -1
    assert _resize_rc(lib, ok, n=0) == -1
    assert _resize_rc(lib, [[0, 10, 20, 59]]) == -1                       # pitch < 3 * w
    assert _resize_rc(lib, [[64, 10, 20, 60]], nbytes=600) == -1          # past the end of the buffer
    assert _resize_rc(lib, [[-16, 10, 20, 60]]) == -1
    assert _resize_rc(lib, ok, params=C.c_void_p((1 << 20) + 4)) == -1    # params not 8-byte aligned


def test_box_kernels_reject_bad_arguments(lib):
    fake = C.c_void_p(1 << 20)
    assert lib.lib.yb_resize_boxes(fake, fake, 1, 4, 3, fake, 32, 32, 1, None) == -1      # box_ld < 4
    assert lib.lib.yb_resize_boxes(fake, fake, 1, 0, 5, fake, 32, 32, 1, None) == -1
    assert lib.lib.yb_resize_boxes(fake, fake, 1, 4, 5, fake, 32, 32, 3, None) == -1
    assert lib.lib.yb_resize_boxes(None, fake, 1, 4, 5, fake, 32, 32, 1, None) == -1
    assert lib.lib.yb_restore_boxes(fake, fake, 0, 4, 4, fake, None) == -1
    assert lib.lib.yb_restore_boxes(fake, fake, 1, 4, 4, None, None) == -1
    assert lib.lib.yb_restore_boxes(fake, fake, 1, 4, 4, C.c_void_p((1 << 20) + 4), None) == -1
