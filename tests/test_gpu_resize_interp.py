"""GPU tests of the training resize (yb_resize_batch_interp, utils.data_aug.resize_train_batch and resize_with_bbox
with interp 2..4): byte for byte against the reference-generated goldens (tests/golden/make_golden_resize_interp.py,
tests/golden/augment.npz) and the numpy restatement (tests/resize_interp_ref.py), which
tests/test_resize_interp_host.py pins to the goldens and to cv2."""
import hashlib
import os

import numpy as np
import pytest
import torch

from tests import resize_interp_cases as K
from tests import resize_interp_ref as M
from tests import resize_ref as R
from tests.test_augment_host import golden_inputs, seed_golden

pytestmark = pytest.mark.gpu


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "resize_interp.npz"))


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _bgr_u8(x):
    """float32 RGB / 255 on the device -> the uint8 BGR image it was made from."""
    return np.rint(x.cpu().numpy()[..., ::-1].astype(np.float64) * 255).astype(np.uint8)


def _params(img, nw, nh, letterbox):
    h, w = img.shape[:2]
    if letterbox:
        ratio, _, _, dw, dh = R.letterbox_geometry(h, w, nw, nh)
        return [ratio, float(dw), float(dh), 1.0]
    return [w / float(nw), h / float(nh), 0.0, 0.0]


def test_golden_cases_bit_exact(golden_dir):
    from yolov3_tensorflow_b200.utils import data_aug as A
    g = _golden(golden_dir)
    sha = dict(zip(g["keys"].tolist(), g["sha256"].tolist()))
    for i, (sh, sw, nw, nh), full in K.cases():
        src = K.source(i, (sh, sw))
        for interp in K.INTERPS:
            for lb in (True, False):
                key = f"{'lb' if lb else 'st'}{interp}_{i}"
                x, p = A.resize_train_batch([src], nw, nh, interp, letterbox=lb)
                assert tuple(x.shape) == (1, nh, nw, 3)
                got = _bgr_u8(x[0])
                assert _sha(got) == sha[key], key
                assert np.array_equal(x[0].cpu().numpy(), R.normalize(got)), key     # exactly u8 / 255
                if full:
                    assert np.array_equal(got, g[key]), key
                assert p[0].cpu().tolist() == _params(src, nw, nh, lb), key


def test_resize_with_bbox_equals_reference(golden_dir):
    from yolov3_tensorflow_b200.utils import data_aug as A
    g = _golden(golden_dir)
    for i, (sh, sw, nw, nh), full in K.cases():
        if not full:
            continue
        src, gt = K.source(i, (sh, sw)), K.boxes(i, sh, sw)
        for interp in K.INTERPS:
            for lb in (True, False):
                key = f"{'lb' if lb else 'st'}{interp}_{i}"
                x, b = A.resize_with_bbox(src, gt.copy(), nw, nh, interp=interp, letterbox=lb)
                assert np.array_equal(x.cpu().numpy(), R.normalize(g[key])), key
                assert np.array_equal(b.cpu().numpy(), g[f"box_{key}"]), key
                if interp == 2:                              # cv2 with Intel IPP (its default): within 1
                    d = np.abs(_bgr_u8(x).astype(np.int16) - g[f"ipp_{key}"].astype(np.int16))
                    assert d.max() <= 1, key


def _mixed_images():
    imgs = [K.source(i, c[:2]) for i, c, _ in K.cases()]
    rng = np.random.default_rng(3)
    imgs += [rng.integers(0, 256, s, dtype=np.uint8) for s in ((375, 500, 3), (1, 1, 3), (416, 416, 3), (208, 832, 3),
                                                                (2, 3, 3), (321, 123, 3))]
    return imgs


@pytest.mark.parametrize("size", [(320, 320), (416, 416), (608, 608), (96, 64)])
@pytest.mark.parametrize("letterbox", [True, False])
def test_mixed_interps_in_one_batch(size, letterbox):
    from yolov3_tensorflow_b200.utils import data_aug as A
    nw, nh = size
    imgs = _mixed_images()
    interp = np.arange(len(imgs), dtype=np.int64) % 5
    x, p = A.resize_train_batch(imgs, nw, nh, interp, letterbox=letterbox)
    x, p = x.cpu().numpy(), p.cpu().numpy()
    for i, (img, it) in enumerate(zip(imgs, interp.tolist())):
        want, _ = M.preprocess(img, nw, nh, letterbox, it)
        assert np.array_equal(x[i], want), (i, it)
        assert p[i].tolist() == _params(img, nw, nh, letterbox), i
    for it in (0, 1):                                       # byte-identical to the evaluation path
        rows = [i for i in range(len(imgs)) if interp[i] == it]
        xe, pe = A.preprocess_batch([imgs[i] for i in rows], nw, nh, letterbox=letterbox, interp=it)
        assert np.array_equal(x[rows], xe.cpu().numpy()) and np.array_equal(p[rows], pe.cpu().numpy())


def test_one_interp_for_the_batch_and_out():
    from yolov3_tensorflow_b200.utils import data_aug as A
    imgs = _mixed_images()[:8]
    packed = A.PackedImages(imgs)
    out = torch.full((len(imgs), 64, 80, 3), -1.0, device="cuda")
    for it in range(5):
        x, _ = A.resize_train_batch(packed, 80, 64, it, out=out)
        assert x is out
        for i, img in enumerate(imgs):
            assert np.array_equal(out[i].cpu().numpy(), M.preprocess(img, 80, 64, True, it)[0]), (it, i)
    with pytest.raises(ValueError, match="out must be"):
        A.resize_train_batch(packed, 80, 64, 2, out=out[:, :, :40])
    with pytest.raises(ValueError, match="interp"):
        A.resize_train_batch(packed, 80, 64, 5)


def test_decoded_batch_goes_in_without_upload(golden_dir):
    from yolov3_tensorflow_b200.utils import data_aug as D
    packed = D.decode_jpeg_batch([os.path.join(golden_dir, f) for f in ("dog.jpg", "messi.jpg")] * 3)
    host = [packed.image(i).cpu().numpy() for i in range(packed.n)]
    data_ptr = packed.data.data_ptr()
    interp = np.array([2, 3, 4, 4, 3, 2], np.int64)
    x, _ = D.resize_train_batch(packed, 416, 416, interp)
    assert packed.data.data_ptr() == data_ptr
    for i, (img, it) in enumerate(zip(host, interp.tolist())):
        assert np.array_equal(x[i].cpu().numpy(), M.preprocess(img, 416, 416, True, it)[0]), i


def _subset(packed, keep):
    """The images `keep` of a PackedImages, pixels shared (only a new descriptor table crosses)."""
    from yolov3_tensorflow_b200.utils import data_aug as D
    desc = np.ascontiguousarray(packed.desc[keep])
    head = torch.from_numpy(desc.view(np.uint8).reshape(-1).copy()).to(packed.device)
    return D.PackedImages.from_device(torch.cat([head, packed.pixels]), desc)


def test_augment_resize_flip_chain_equals_reference_golden(golden_dir):
    """augment_train_batch -> resize_train_batch(interp) -> yb_resize_boxes -> flip_batch equals every final_img{i} /
    final_boxes{i} the reference recorded (its INTER_AREA draws included)."""
    from yolov3_tensorflow_b200 import _lib
    from yolov3_tensorflow_b200.utils import data_aug as D
    g = np.load(os.path.join(golden_dir, "augment.npz"))
    imgs, boxes, labels, mix = golden_inputs(g)
    seed_golden()
    packed, bx, _, interp, flip = D.augment_train_batch(imgs, boxes, labels, mix_with=mix)
    keep = [i for i in range(packed.n) if f"final_img{i}" in g.files]
    assert len(keep) == packed.n - 1 and sorted(set(interp[keep].tolist())) == [0, 1, 3]
    sub = _subset(packed, keep)
    S = 64
    x, _ = D.resize_train_batch(sub, S, S, interp[keep], letterbox=True)
    vmax = max(len(bx[i]) for i in keep)
    b = np.zeros((len(keep), vmax, 5), np.float32)
    for k, i in enumerate(keep):
        b[k, :len(bx[i])] = bx[i]
    bd = torch.from_numpy(b).cuda()
    cnt = torch.tensor([len(bx[i]) for i in keep], dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib.yb_resize_boxes(_lib.ptr(bd), _lib.ptr(cnt), len(keep), vmax, 5, _lib.ptr(sub.desc_dev), S, S,
                                        1, _lib.stream_handle()), "yb_resize_boxes")
    D.flip_batch(x, flip[keep], bd, cnt)
    xs, bs = x.cpu().numpy(), bd.cpu().numpy()
    for k, i in enumerate(keep):
        assert np.array_equal(xs[k], R.normalize(g[f"final_img{i}"])), (i, int(interp[i]))
        want = g[f"final_boxes{i}"]
        got = bs[k, :len(want)]
        if want.dtype == np.float32:
            assert np.array_equal(got, want), i
        else:                                        # a mix-up made the reference's boxes float64
            assert np.allclose(got, want, rtol=1e-6, atol=1e-4), i
