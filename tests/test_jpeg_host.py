"""CPU tests of the JPEG decoder: the numpy restatement (tests/jpeg_ref.py) equals every golden and live cv2, and
the host side of the C ABI (yb_jpeg_parse, pack, argument checks) needs no device."""
import ctypes as C

import numpy as np
import pytest

from tests import jpeg_ref as R
from tests.jpeg_cases import load, sha, demo


META, CASES = load()


@pytest.mark.parametrize("case", [c for c in CASES if c["note"] in ("synthetic", "orientation", "divergent")],
                         ids=lambda c: c["name"])
def test_restatement_equals_golden(case):
    out, st = R.decode(case["data"])
    assert st == 0
    assert list(out.shape) == case["shape"] and sha(out) == case["sha256"]
    if "expect" in case:
        assert np.array_equal(out, case["expect"])


@pytest.mark.parametrize("case", [c for c in CASES if c["note"] == "corrupt"], ids=lambda c: c["name"])
def test_restatement_flags_corrupt(case):
    _, st = R.decode(case["data"])
    assert st == case["status"] != 0


def test_corrupt_fixtures_cover_every_status():
    bits = 0
    for c in CASES:
        bits |= c["status"]
    assert bits == R.BAD_MARKER | R.BAD_RST | R.BAD_CODE | R.BAD_INDEX | R.TRUNCATED
    # a bad code alone is not also reported as truncated data
    assert any(c["status"] == R.BAD_CODE for c in CASES) and any(c["status"] == R.BAD_INDEX for c in CASES)


@pytest.mark.parametrize("name", ["dog.jpg", "messi.jpg"])
def test_restatement_equals_demo(name):
    out, st = R.decode(demo(name))
    assert st == 0 and list(out.shape) == META[name]["shape"] and sha(out) == META[name]["sha256"]


def test_restatement_equals_live_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    samp = [cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
            cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420]
    for it in range(300):
        h, w = int(rng.integers(1, 48)), int(rng.integers(1, 48))
        kind = it % 3
        if kind == 0:
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        elif kind == 1:
            img = np.clip(np.add.outer(np.arange(h) * 9, np.arange(w) * 4)[:, :, None] + rng.integers(0, 99, 3),
                          0, 255).astype(np.uint8)
        else:
            img = np.full((h, w, 3), rng.integers(0, 256, 3), np.uint8)
        if it % 7 == 0:
            img = img[:, :, 1].copy()
        q = 100 if it % 5 == 0 else int(rng.integers(10, 101))
        ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                             samp[it % 4], cv2.IMWRITE_JPEG_RST_INTERVAL, int(rng.choice([0, 1, 3, 7])),
                                             cv2.IMWRITE_JPEG_OPTIMIZE, it % 2])
        out, st = R.decode(enc.tobytes())
        ref = cv2.imdecode(enc, cv2.IMREAD_COLOR)
        assert st == 0 and np.array_equal(out, ref), (it, h, w, q)


def test_parse_reports_header():
    from yolov3_tensorflow_b200.utils.data_aug import jpeg_info
    for name, (hs, vs, ri) in (("dog.jpg", (1, 2, 96)), ("messi.jpg", (2, 2, 0))):
        info = jpeg_info(demo(name))
        assert (info["height"], info["width"], 3) == tuple(META[name]["shape"])
        assert (info["h_samp"], info["v_samp"], info["restart_interval"], info["components"]) == (hs, vs, ri, 3)
    for c in CASES:
        if c["name"].startswith("exif_"):
            o = int(c["name"][5:])
            info = jpeg_info(c["data"])
            assert info["orientation"] == o and [info["height"], info["width"]] == c["shape"][:2]
        elif c["note"] == "rejected":
            with pytest.raises(ValueError, match=c["reason"]):
                jpeg_info(c["data"])
        elif "grey" in c["name"]:
            assert jpeg_info(c["data"])["components"] == 1
    with pytest.raises(ValueError, match="no SOI"):
        jpeg_info(b"\x89PNG....")
    with pytest.raises(ValueError, match="truncated header"):
        jpeg_info(demo("dog.jpg")[:300])


def test_pack_names_the_image_and_abi_checks_arguments():
    from yolov3_tensorflow_b200 import _lib
    lib = _lib.lib
    good, bad = demo("dog.jpg"), [c for c in CASES if c["name"] == "progressive"][0]["data"]
    files = [good, bad]
    ptrs = (C.c_void_p * 2)(*[C.cast(C.c_char_p(f), C.c_void_p) for f in files])
    sizes = (C.c_size_t * 2)(*[len(f) for f in files])
    n = C.c_size_t()
    assert lib.yb_jpeg_pack_bytes(ptrs, sizes, 2, C.byref(n)) == -3
    assert b"image 1: progressive" in lib.yb_last_error_string()
    assert lib.yb_jpeg_pack_bytes(ptrs, sizes, 1, C.byref(n)) == 0 and n.value > 0
    blob = (C.c_uint8 * n.value)()
    desc = np.zeros((1, 4), np.int64)
    assert lib.yb_jpeg_pack(ptrs, sizes, 1, blob, n.value - 1, None) == -1
    assert lib.yb_jpeg_pack(ptrs, sizes, 1, blob, n.value, desc.ctypes.data_as(C.c_void_p)) == 0
    assert desc.tolist() == [[0, 576, 768, 3 * 768]]
    ws, pix = C.c_size_t(), C.c_size_t()
    assert lib.yb_jpeg_workspace_bytes(blob, 2, C.byref(ws), None) == -1
    assert lib.yb_jpeg_workspace_bytes(blob, 1, C.byref(ws), C.byref(pix)) == 0 and pix.value == 576 * 768 * 3
    # argument errors return before any device work (no device here)
    assert lib.yb_jpeg_decode(None, blob, 1, None, None, None, None, 0, None) == -1
    fake = C.c_void_p(16)
    assert lib.yb_jpeg_decode(fake, blob, 1, fake, fake, fake, fake, ws.value - 1, None) == -4
    assert lib.yb_jpeg_decode(fake, None, 1, fake, fake, fake, fake, ws.value, None) == -1
    _lib.set_option("YB_JPEG_SUBSEQ_BITS", 48)
    try:
        assert lib.yb_jpeg_pack_bytes(ptrs, sizes, 1, C.byref(n)) == -1
    finally:
        _lib.set_option("YB_JPEG_SUBSEQ_BITS", None)


def test_pack_rejects_streams_past_32_bit_positions():
    """Each restart segment starts on a subsequence boundary: 65,536 one-MCU segments at 65,536-bit subsequences
    need 2^32 stream bits, which the 32-bit bit positions cannot address."""
    cv2 = pytest.importorskip("cv2")
    from yolov3_tensorflow_b200 import _lib
    ok, enc = cv2.imencode(".jpg", np.full((2048, 2048, 3), 90, np.uint8),
                           [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444,
                            cv2.IMWRITE_JPEG_RST_INTERVAL, 1])
    f = enc.tobytes()
    ptrs, sizes, n = (C.c_void_p * 1)(C.cast(C.c_char_p(f), C.c_void_p)), (C.c_size_t * 1)(len(f)), C.c_size_t()
    assert _lib.lib.yb_jpeg_pack_bytes(ptrs, sizes, 1, C.byref(n)) == 0
    _lib.set_option("YB_JPEG_SUBSEQ_BITS", 65536)
    try:
        assert _lib.lib.yb_jpeg_pack_bytes(ptrs, sizes, 1, C.byref(n)) == -3
        assert b"image 0" in _lib.lib.yb_last_error_string() and b"2^32" in _lib.lib.yb_last_error_string()
    finally:
        _lib.set_option("YB_JPEG_SUBSEQ_BITS", None)
