"""CPU tests of the JPEG encoder: the numpy restatement (tests/jpeg_enc_ref.py) equals every golden and live
cv2.imencode on 300 seeded random cases; the C-ABI header builder equals the golden headers; argument validation
returns the documented status codes; unsupported requests raise ValueError."""
import ctypes as C

import numpy as np
import pytest

from tests import jpeg_enc_cases as E
from tests import jpeg_enc_ref as R

META, CASES = E.load()


def test_fixture_records_versions():
    assert META["opencv"] == "4.13.0" and META["libjpeg_turbo"].startswith("3.1")
    assert len(CASES) >= 90


@pytest.mark.parametrize("k", range(len(CASES)))
def test_restatement_equals_golden(k):
    c = CASES[k]
    out = R.encode(E.image(c), **c["kw"])
    assert E.matches(c, out["data"]), c["name"]
    assert int(np.ceil(out["bits"].sum() / 8)) <= len(out["data"])


def _random_case(rng):
    h, w = int(rng.integers(1, 80)), int(rng.integers(1, 80))
    kind = ["noise", "gradient", "flat", "dog.jpg", "messi.jpg"][int(rng.integers(0, 5))]
    if kind.endswith(".jpg"):
        h, w = int(rng.integers(1, 300)), int(rng.integers(1, 300))
    c = dict(h=h, w=w, kind=kind, grey=bool(rng.random() < 0.2), seed=int(rng.integers(0, 1 << 30)))
    kw = dict(quality=int(rng.integers(-5, 106)), sampling=str(rng.choice(list(R.SAMPLING))),
              restart_interval=int(rng.choice([0, 0, 1, 2, 3, 7, 50])))
    if rng.random() < 0.3:
        kw["luma_quality"] = int(rng.integers(-1, 105))
        if rng.random() < 0.7:
            kw["chroma_quality"] = int(rng.integers(-1, 105))
    elif rng.random() < 0.1:
        kw["chroma_quality"] = int(rng.integers(0, 101))
    return c, kw


def test_restatement_equals_live_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(2026)
    bad = []
    for i in range(300):
        c, kw = _random_case(rng)
        img = E.image(c)
        ref = cv2.imencode(".jpg", img, R.cv2_params(**kw))[1].tobytes()
        if R.encode(img, **kw)["data"] != ref:
            bad.append((i, img.shape, kw))
    assert not bad, bad[:5]


def test_bgr_and_rgb_order_give_the_same_file():
    """OpenCV hands BGR to libjpeg (JCS_EXT_BGR); converting to RGB first and encoding as RGB must not change the
    file: the restatement's colour conversion reads B, G, R by position."""
    cv2 = pytest.importorskip("cv2")
    img = E.image(dict(h=37, w=51, kind="messi.jpg", grey=False, seed=4))
    assert R.encode(img)["data"] == cv2.imencode(".jpg", img, R.cv2_params())[1].tobytes()
    y, cb, cr = R.rgb_to_ycc(img)
    y2, cb2, cr2 = R.rgb_to_ycc(cv2.cvtColor(cv2.cvtColor(img, cv2.COLOR_BGR2RGB), cv2.COLOR_RGB2BGR))
    assert np.array_equal(y, y2) and np.array_equal(cb, cb2) and np.array_equal(cr, cr2)


def _image(h, w, channels=3, **kw):
    from yolov3_tensorflow_b200 import _lib
    args = dict(quality=95, luma_quality=-1, chroma_quality=-1, sampling="420", restart_interval=0)
    args.update(kw)
    return _lib.JpegEncImage(0x1000, w * channels, h, w, channels, args["quality"], args["luma_quality"],
                             args["chroma_quality"], _lib.YB_JPEG_SAMPLING.get(args["sampling"], 7),
                             args["restart_interval"])


def _header(im):
    from yolov3_tensorflow_b200 import _lib
    n = C.c_size_t()
    assert _lib.lib.yb_jpeg_enc_header(C.byref(im), None, 0, C.byref(n)) == 0
    buf = (C.c_uint8 * n.value)()
    assert _lib.lib.yb_jpeg_enc_header(C.byref(im), buf, n.value, C.byref(n)) == 0
    return bytes(buf)


@pytest.mark.parametrize("k", range(len(CASES)))
def test_cabi_header_equals_golden(k):
    c = CASES[k]
    kw = dict(c["kw"])
    kw.setdefault("sampling", "420")
    for key in ("luma_quality", "chroma_quality"):
        if kw.get(key) is None:
            kw[key] = -1
    hdr = _header(_image(c["h"], c["w"], 1 if c["grey"] else 3, **kw))
    assert hdr == R.header(c["h"], c["w"], 1 if c["grey"] else 3, **c["kw"])
    if "data" in c:
        assert c["data"].startswith(hdr)


def test_cabi_status_codes():
    from yolov3_tensorflow_b200 import _lib
    L = _lib.lib
    n = C.c_size_t()
    ok = _image(16, 16)
    assert L.yb_jpeg_enc_header(None, None, 0, C.byref(n)) == -1
    assert L.yb_jpeg_enc_header(C.byref(_image(0, 5)), None, 0, C.byref(n)) == -1
    assert b"outside 1..65535" in L.yb_last_error_string()
    assert L.yb_jpeg_enc_header(C.byref(_image(5, 65536)), None, 0, C.byref(n)) == -1
    assert L.yb_jpeg_enc_header(C.byref(_image(5, 5, channels=2)), None, 0, C.byref(n)) == -1
    assert b"channels" in L.yb_last_error_string()
    assert L.yb_jpeg_enc_header(C.byref(_image(5, 5, sampling="bad")), None, 0, C.byref(n)) == -1
    assert b"sampling" in L.yb_last_error_string()
    small = (C.c_uint8 * 10)()
    assert L.yb_jpeg_enc_header(C.byref(ok), small, 10, C.byref(n)) == -4 and n.value > 10
    ims = (_lib.JpegEncImage * 3)(_image(8, 8), _image(65535, 65535), _image(4, 4, channels=4))
    assert L.yb_jpeg_enc_pack_bytes(ims, 3, C.byref(n)) == -1
    assert L.yb_last_error_string().startswith(b"image 2: ")
    ims[2] = _image(4, 4, channels=1)
    ims[1].pixels = None
    assert L.yb_jpeg_enc_pack_bytes(ims, 3, C.byref(n)) == -1
    assert L.yb_last_error_string().startswith(b"image 1: null pixels")
    ims[1] = _image(65535, 65535)
    assert L.yb_jpeg_enc_pack_bytes(ims, 0, C.byref(n)) == -1
    assert L.yb_jpeg_enc_pack_bytes(ims, 3, C.byref(n)) == 0
    blob = (C.c_uint8 * n.value)()
    assert L.yb_jpeg_enc_pack(ims, 3, blob, n.value - 16) == -1
    assert L.yb_jpeg_enc_pack(ims, 3, blob, n.value) == 0
    ws, out = C.c_size_t(), C.c_size_t()
    assert L.yb_jpeg_enc_workspace_bytes(blob, 2, C.byref(ws), C.byref(out)) == -1
    assert L.yb_jpeg_enc_workspace_bytes(blob, 3, C.byref(ws), C.byref(out)) == 0
    assert out.value > 65535 * 65535 * 3 // 2 and ws.value > out.value // 2
    assert L.yb_jpeg_enc_workspace_bytes((C.c_uint8 * 64)(), 3, C.byref(ws), None) == -1
    assert b"yb_jpeg_enc_pack" in L.yb_last_error_string()
    assert L.yb_jpeg_enc_encode(blob, blob, 3, None, 0, None, None, 0, None) == -1


def test_python_rejections_name_image_and_reason():
    from yolov3_tensorflow_b200.utils.data_aug import encode_jpeg_batch
    good = np.zeros((8, 8, 3), np.uint8)
    with pytest.raises(ValueError, match="progressive"):
        encode_jpeg_batch([good], progressive=True)
    with pytest.raises(ValueError, match="IMWRITE_JPEG_OPTIMIZE"):
        encode_jpeg_batch([good], optimize=True)
    with pytest.raises(ValueError, match="image 1: expected uint8"):
        encode_jpeg_batch([good, good.astype(np.float32)])
    with pytest.raises(ValueError, match="image 0: expected uint8"):
        encode_jpeg_batch([np.zeros((8, 8, 4), np.uint8)])
    with pytest.raises(ValueError, match="image 0: expected uint8"):
        encode_jpeg_batch([np.zeros((8,), np.uint8)])
    with pytest.raises(ValueError, match="image 0: size 0 x 8"):
        encode_jpeg_batch([np.zeros((0, 8, 3), np.uint8)])
    with pytest.raises(ValueError, match="no images"):
        encode_jpeg_batch([])
