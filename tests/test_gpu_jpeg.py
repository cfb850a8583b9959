"""GPU tests of decode_jpeg_batch / yb_jpeg_decode: every golden bit for bit (located stage by stage against
tests/jpeg_ref.py on a mismatch), batches equal single decodes, the subsequence size does not change bytes, corrupt
images get their status and stay in their slot, and the decoded batch feeds preprocess_batch / val_batch / detect_raw
exactly as the cv2 arrays do."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import jpeg_ref as R
from tests.jpeg_cases import load, sha, demo

pytestmark = pytest.mark.gpu
META, CASES = load()
GOOD = [c for c in CASES if c["note"] in ("synthetic", "orientation", "divergent")]
CORRUPT = [c for c in CASES if c["note"] == "corrupt"]


def _decode(files, **kw):
    from yolov3_tensorflow_b200.utils.data_aug import decode_jpeg_batch
    return decode_jpeg_batch(files, **kw)


def _locate(data, got):
    """On a mismatch: the first stage of the restatement the device output disagrees with."""
    st = R.decode(data, stages=True)
    d = np.argwhere(got != st["out"])
    return f"{len(d)} bytes differ, first at {d[0].tolist() if len(d) else None}; restatement status {st['status']}"


def test_goldens_decode_bit_exact():
    p = _decode([c["data"] for c in GOOD])
    assert (p.status.cpu().numpy() == 0).all()
    for i, c in enumerate(GOOD):
        got = p.image(i).cpu().numpy()
        assert list(got.shape) == c["shape"], c["name"]
        assert sha(got) == c["sha256"], f"{c['name']}: {_locate(c['data'], got)}"


@pytest.mark.parametrize("name", ["dog.jpg", "messi.jpg"])
def test_demo_images(name):
    p = _decode([demo(name)])
    got = p.image(0).cpu().numpy()
    assert list(got.shape) == META[name]["shape"]
    assert sha(got) == META[name]["sha256"], _locate(demo(name), got)


def test_batch_of_64_equals_single_decodes_and_desc():
    rng = np.random.default_rng(5)
    pool = GOOD + [dict(data=demo("dog.jpg")), dict(data=demo("messi.jpg"))]
    files = [pool[i]["data"] for i in rng.integers(0, len(pool), 64)]
    p = _decode(files)
    assert np.array_equal(p.desc_dev.view(torch.int64).view(64, 4).cpu().numpy(), p.desc)
    for i, f in enumerate(files):
        assert torch.equal(p.image(i), _decode([f]).image(0))


@pytest.mark.parametrize("bits", [32, 65536])
def test_subsequence_size_does_not_change_bytes(bits):
    from yolov3_tensorflow_b200 import _lib
    files = [c["data"] for c in GOOD[::3]] + [demo("messi.jpg"), demo("dog.jpg")]
    ref = _decode(files)
    _lib.set_option("YB_JPEG_SUBSEQ_BITS", bits)
    try:
        p = _decode(files)
    finally:
        _lib.set_option("YB_JPEG_SUBSEQ_BITS", None)
    assert (p.status.cpu() == 0).all()
    for i in range(len(files)):   # the alignment gaps between slots are not written
        assert torch.equal(p.image(i), ref.image(i))


def test_corrupt_images_status_slot_and_neighbours():
    from yolov3_tensorflow_b200 import _lib
    lib = _lib.lib
    files = []
    for c in CORRUPT:
        files += [GOOD[len(files) % len(GOOD)]["data"], c["data"]]
    n = len(files)
    bufs = [C.create_string_buffer(f, len(f)) for f in files]
    ptrs = (C.c_void_p * n)(*[C.cast(b, C.c_void_p) for b in bufs])
    sizes = (C.c_size_t * n)(*[len(f) for f in files])
    nb = C.c_size_t()
    assert lib.yb_jpeg_pack_bytes(ptrs, sizes, n, C.byref(nb)) == 0
    host = torch.empty((nb.value,), dtype=torch.uint8).pin_memory()
    desc = np.zeros((n, 4), np.int64)
    assert lib.yb_jpeg_pack(ptrs, sizes, n, C.c_void_p(host.data_ptr()), nb.value, desc.ctypes.data_as(C.c_void_p)) == 0
    ws, pix = C.c_size_t(), C.c_size_t()
    assert lib.yb_jpeg_workspace_bytes(C.c_void_p(host.data_ptr()), n, C.byref(ws), C.byref(pix)) == 0
    blob = host.cuda()
    wsb = torch.empty((ws.value,), dtype=torch.uint8, device="cuda")
    out = torch.full((pix.value + 64,), 0xA5, dtype=torch.uint8, device="cuda")   # sentinel everywhere
    dd = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    status = torch.empty((n,), dtype=torch.int32, device="cuda")
    assert lib.yb_jpeg_decode(_lib.ptr(blob), C.c_void_p(host.data_ptr()), n, _lib.ptr(out), _lib.ptr(dd),
                              _lib.ptr(status), _lib.ptr(wsb), ws.value, _lib.stream_handle()) == 0
    st = status.cpu().numpy()
    o = out.cpu().numpy()
    inside = np.zeros(o.size, bool)
    for i in range(n):
        off, h, w, pitch = desc[i]
        inside[off:off + h * pitch] = True
        if i % 2:
            assert st[i] == CORRUPT[i // 2]["status"], CORRUPT[i // 2]["name"]
        else:
            assert st[i] == 0
            assert sha(o[off:off + h * pitch].reshape(h, w, 3)) == GOOD[(i // 2 * 2) % len(GOOD)]["sha256"]
    assert (o[~inside] == 0xA5).all(), "bytes written outside the image slots"
    with pytest.raises(ValueError, match="image 1"):
        _decode(files[:2])


def test_check_false_does_not_sync():
    files = [demo("messi.jpg")] * 8
    _decode(files, check=False)
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)            # keep the stream busy: a sync would wait for it
    ev = torch.cuda.Event()
    ev.record()
    p = _decode(files, check=False)
    assert not ev.query(), "decode_jpeg_batch(check=False) waited for the stream"
    torch.cuda.synchronize()
    assert (p.status.cpu() == 0).all()


def test_decoded_batch_feeds_preprocess_val_and_detect():
    from oracle import yolov3_oracle as O
    import yolov3_tensorflow_b200 as pkg
    from yolov3_tensorflow_b200.utils.data_aug import preprocess_batch
    from yolov3_tensorflow_b200.utils.data_utils import val_batch
    files = [demo("dog.jpg"), demo("messi.jpg")] + [c["data"] for c in GOOD if c["shape"][0] >= 127][:6]
    p = _decode(files)
    arrays = [p.image(i).cpu().numpy() for i in range(len(files))]
    x1, pr1 = preprocess_batch(p, 416, 416)
    x2, pr2 = preprocess_batch(arrays, 416, 416)
    assert torch.equal(x1, x2) and torch.equal(pr1, pr2)
    boxes = [np.array([[10, 10, 60, 80]], np.float32)] * len(files)
    labels = [np.array([3])] * len(files)
    v1 = val_batch(p, boxes, labels, [416, 416], 80, O.COCO_ANCHORS)
    v2 = val_batch(arrays, boxes, labels, [416, 416], 80, O.COCO_ANCHORS)
    for a, b in zip(v1, v2):
        assert torch.equal(a, b)
    m = pkg.yolov3(80, O.COCO_ANCHORS, dtype="fp16")
    m.set_params(O.make_params(80, seed=3, random_bn=True, det_scale=8.0, conf_bias=-2.0), "HWIO")
    d1 = m.detect_raw(x1)
    d2 = m.detect_raw(x2)
    assert torch.equal(d1[5], d2[5])
    for i, k in enumerate(d1[5].tolist()):
        for a, b in zip(d1[1:5], d2[1:5]):
            assert torch.equal(a[i, :k], b[i, :k])
