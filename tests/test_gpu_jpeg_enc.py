"""GPU tests of encode_jpeg_batch / yb_jpeg_enc_encode: every golden byte for byte (a mismatch is located block by
block against tests/jpeg_enc_ref.py), a mixed batch of 64 against single encodes, host / CUDA / PackedImages
sources, decode -> encode without the pixels leaving the device, the device round trip, and to_host=False without
a host synchronisation."""
import numpy as np
import pytest
import torch

from tests import jpeg_enc_cases as E
from tests import jpeg_enc_ref as R

pytestmark = pytest.mark.gpu

META, CASES = E.load()


def _encode(images, **kw):
    from yolov3_tensorflow_b200.utils.data_aug import encode_jpeg_batch
    return encode_jpeg_batch(images, **kw)


_DEFAULTS = dict(quality=95, sampling="420", restart_interval=0, luma_quality=None, chroma_quality=None)


def _kwargs(cases):
    """Per-image argument lists of encode_jpeg_batch for these cases."""
    return {a: [c["kw"].get(a, d) for c in cases] for a, d in _DEFAULTS.items()}


def _locate(img, kw, got):
    """On a mismatch: the first block whose bits the device file disagrees with, per the restatement."""
    st = R.encode(img, **kw)
    ref = st["data"]
    hdr = len(st["header"])
    if got[:hdr] != ref[:hdr]:
        return "header differs"
    i = next((k for k in range(min(len(got), len(ref))) if got[k] != ref[k]), min(len(got), len(ref)))
    # map the first differing stuffed byte back to a bit of the unstuffed stream, then to its block
    body = ref[hdr:i]
    unstuffed = len(body.replace(b"\xff\x00", b"\xff")) * 8
    ends = np.cumsum(st["bits"])
    b = int(np.searchsorted(ends, unstuffed, side="right"))
    return (f"{len(got)} vs {len(ref)} bytes, first difference at byte {i}: block {b} (component "
            f"{int(st['comp'][min(b, len(ends) - 1)])}, dummy {bool(st['dummy'][min(b, len(ends) - 1)])}) "
            "(with restart markers the block is approximate)")


def test_goldens_byte_exact():
    imgs = [E.image(c) for c in CASES]
    out = []
    for k in range(0, len(CASES), 32):            # the goldens in batches, each case with its own arguments
        chunk = CASES[k:k + 32]
        out += _encode(imgs[k:k + 32], **_kwargs(chunk))
    for c, img, got in zip(CASES, imgs, out):
        assert E.matches(c, got), f"{c['name']}: {_locate(img, c['kw'], got)}"


def test_batch_of_64_mixed_equals_single_encodes():
    rng = np.random.default_rng(64)
    pick = [CASES[i] for i in rng.integers(0, len(CASES), 64)]
    imgs = [E.image(c) for c in pick]
    # half the images already on the device, half on the host
    srcs = [torch.from_numpy(im).cuda() if i % 2 else im for i, im in enumerate(imgs)]
    batch = _encode(srcs, **_kwargs(pick))
    for i, (c, im) in enumerate(zip(pick, imgs)):
        single = _encode([im], **c["kw"])[0]
        assert batch[i] == single, f"image {i} ({c['name']})"
        assert E.matches(c, single), c["name"]


def test_decode_then_encode_stays_on_device():
    from yolov3_tensorflow_b200.utils.data_aug import decode_jpeg_batch
    files = []
    for name in ("dog.jpg", "messi.jpg"):
        with open(f"{E.GOLDEN}/{name}", "rb") as f:
            files.append(f.read())
    packed = decode_jpeg_batch(files)
    for kw in (dict(quality=95), dict(quality=75), dict(quality=90, sampling="444", restart_interval=3)):
        got = _encode(packed, **kw)
        for name, g in zip(("dog.jpg", "messi.jpg"), got):
            c = next(c for c in CASES if c.get("whole") and c["kind"] == name and c["kw"] == kw)
            assert E.matches(c, g), f"{name} {kw}"


def test_device_round_trip_equals_cv2_imdecode_of_imencode():
    from yolov3_tensorflow_b200.utils.data_aug import decode_jpeg_batch
    cases = [c for c in CASES if c["kw"].get("sampling") != "411" and not c.get("whole")]
    files = _encode([E.image(c) for c in cases], **_kwargs(cases))
    packed = decode_jpeg_batch(files)
    for i, c in enumerate(cases):
        assert E.sha(packed.image(i).cpu().numpy()) == c["roundtrip_sha256"], c["name"]


def test_cuda_tensor_sources_and_grey_shapes():
    c = next(c for c in CASES if c["grey"] and c["h"] >= 16 and c["w"] >= 16)
    g = E.image(c)
    variants = [g, g[:, :, None], torch.from_numpy(g).cuda(), torch.from_numpy(g[:, :, None]).cuda()]
    for got in _encode(variants, **c["kw"]):
        assert E.matches(c, got)


def test_to_host_false_does_not_sync_and_matches():
    imgs = [E.image(c) for c in CASES if c["kind"] == "dog.jpg" and c["h"] == 375][:1] * 8
    ref = _encode(imgs)
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)            # keep the stream busy: a sync would wait for it
    ev = torch.cuda.Event()
    ev.record()
    data, desc = _encode(imgs, to_host=False)
    assert not ev.query(), "encode_jpeg_batch(to_host=False) waited for the stream"
    torch.cuda.synchronize()
    d = desc.cpu().numpy()
    assert d.shape == (8, 2) and d[0, 0] == 0 and (d[1:, 0] == d[:-1, 0] + d[:-1, 1]).all()
    host = data.cpu().numpy()
    assert [host[o: o + n].tobytes() for o, n in d.tolist()] == ref


def test_write_jpeg_batch(tmp_path):
    from yolov3_tensorflow_b200.utils.data_aug import write_jpeg_batch
    cs = [c for c in CASES if "data" in c][:3]
    paths = [str(tmp_path / f"{k}.jpg") for k in range(3)]
    write_jpeg_batch(paths, [E.image(c) for c in cs], **_kwargs(cs))
    for p, c in zip(paths, cs):
        with open(p, "rb") as f:
            assert f.read() == c["data"]
