"""utils/data_aug.py of the reference, the functions on the inference and evaluation input path: `letterbox_resize`
(:274-293) and `resize_with_bbox` (:296-318), fused with the caller's BGR->RGB + float32 / 255
(test_single_image.py:44-46) into device kernels (libyolob200.so: yb_letterbox_normalize for one image, yb_resize_batch
for a batch of images of different sizes, letterbox or stretch, nearest or bilinear; yb_resize_batch_interp for the
training resize with every cv2.resize interpolation of the reference, 0..4, one per image), plus the detections' way
back to the source image (test_single_image.py:64-70, yb_restore_boxes).  Bit-exact vs cv2.resize of OpenCV 4.13
(INTER_CUBIC: OpenCV's own code, within 1 of its Intel IPP dispatch).  The training augmentations around the resize (`mix_up`, `random_color_distort`, `random_expand`,
`random_crop_with_constraints`, `random_flip`, batched as `augment_train_batch` + `flip_batch`) draw on the host in the
reference's order and run as device kernels (yb_augment_batch, yb_flip_batch).  `decode_jpeg_batch` replaces
the cv2.imread in front of them (utils/data_utils.py:130, test_single_image.py:38): baseline JPEG files decoded on the
device (yb_jpeg_decode), equal to cv2.imread byte for byte, straight into the PackedImages layout.
`encode_jpeg_batch` / `write_jpeg_batch` are cv2.imencode('.jpg') / cv2.imwrite (test_single_image.py:85) for a batch
on the device (yb_jpeg_enc_encode), byte for byte."""
from __future__ import annotations

import ctypes as C
import random

import numpy as np
import torch

from .. import _lib
from .._lib import lib, check, ptr, stream_handle


def letterbox_params(ori_height, ori_width, new_width, new_height):
    """(resize_ratio, resize_w, resize_h, dw, dh) of letterbox_resize — what test_single_image.py:64-66 needs to map
    the detections back to the original image."""
    ratio = C.c_double()
    rh, rw, dh, dw = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    check(lib.yb_letterbox_params(int(ori_height), int(ori_width), int(new_height), int(new_width), C.byref(ratio),
                                  C.byref(rh), C.byref(rw), C.byref(dh), C.byref(dw)), "yb_letterbox_params")
    return ratio.value, rw.value, rh.value, dw.value, dh.value


def letterbox_preprocess(img_bgr, new_width, new_height, device=None, out=None):
    """img_bgr: uint8 [H, W, 3] in OpenCV's BGR order (numpy array or torch tensor, host or CUDA) ->
    (x float32 [1, new_height, new_width, 3] RGB in [0, 1] on the device, resize_ratio, dw, dh):
    letterbox_resize(img, new_width, new_height) + cvtColor(BGR2RGB) + np.float32 + / 255. of the reference."""
    dev = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
    t = torch.from_numpy(np.ascontiguousarray(img_bgr)) if isinstance(img_bgr, np.ndarray) else img_bgr
    if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3:
        raise ValueError(f"letterbox_preprocess expects a uint8 [H, W, 3] image, got {t.dtype} {tuple(t.shape)}")
    t = t.to(dev, non_blocking=True).contiguous()
    h, w = int(t.shape[0]), int(t.shape[1])
    ratio, rw, rh, dw, dh = letterbox_params(h, w, new_width, new_height)
    if out is None:
        out = torch.empty((1, int(new_height), int(new_width), 3), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        check(lib.yb_letterbox_normalize(ptr(t), h, w, 3 * w, int(new_height), int(new_width), ptr(out), stream_handle()),
              "yb_letterbox_normalize")
    return out, ratio, dw, dh


class PackedImages:
    """A batch of uint8 BGR images of any sizes on the device: `data` holds the int64 [n, 4] descriptor table
    (byte offset, h, w, row pitch) followed by the pixels, `desc` is the host copy of the table."""

    def __init__(self, images, device=None):
        dev = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        arrs = []
        for i, im in enumerate(images):
            a = im.detach().cpu().numpy() if isinstance(im, torch.Tensor) else np.asarray(im)
            if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
                raise ValueError(f"image {i}: expected a uint8 [H, W, 3] BGR image, got {a.dtype} {a.shape}")
            arrs.append(a)
        n = len(arrs)
        if n == 0:
            raise ValueError("no images")
        desc = np.zeros((n, 4), np.int64)
        off = 0
        for i, a in enumerate(arrs):
            h, w = a.shape[:2]
            desc[i] = (off, h, w, 3 * w)
            off += (a.size + 15) // 16 * 16
        head = n * 32
        pinned = torch.empty((head + max(off, 1),), dtype=torch.uint8, pin_memory=True)
        buf = pinned.numpy()
        buf[:head] = desc.view(np.uint8).reshape(-1)
        for (o, _, _, _), a in zip(desc.tolist(), arrs):
            buf[head + o: head + o + a.size] = a.reshape(-1)
        self.device = dev
        self.n = n
        self.desc = desc
        self.data = pinned.to(dev, non_blocking=True)          # the one host -> device copy
        self.h2d_bytes = int(pinned.numel())
        self.status = None

    @classmethod
    def from_device(cls, data, desc, status=None, h2d_bytes=0):
        """A batch whose pixels are already on the device: data uint8 CUDA tensor holding the int64 [n, 4]
        descriptor table and the pixels (the layout above), desc its int64 [n, 4] host copy.  No copy is made."""
        self = cls.__new__(cls)
        self.device = data.device
        self.desc = np.ascontiguousarray(desc, np.int64)
        self.n = int(self.desc.shape[0])
        self.data = data
        self.h2d_bytes = int(h2d_bytes)
        self.status = status
        return self

    def __len__(self):
        return self.n

    def image(self, i):
        """uint8 [H, W, 3] BGR view of image i on the device."""
        off, h, w, pitch = (int(v) for v in self.desc[i])
        return self.pixels[off: off + h * pitch].view(h, w, 3)

    @property
    def desc_dev(self):
        return self.data[: self.n * 32]

    @property
    def pixels(self):
        return self.data[self.n * 32:]


def _resize_packed(packed, new_width, new_height, letterbox, interp, out=None):
    n, dev = packed.n, packed.device
    new_w, new_h = int(new_width), int(new_height)
    if out is None:
        out = torch.empty((n, new_h, new_w, 3), dtype=torch.float32, device=dev)
    elif (out.dtype != torch.float32 or tuple(out.shape) != (n, new_h, new_w, 3) or not out.is_contiguous()
          or out.device != dev):
        raise ValueError(f"out must be a contiguous float32 [{n}, {new_h}, {new_w}, 3] tensor on {dev}")
    params = torch.empty((n, 4), dtype=torch.float64, device=dev)
    desc = np.ascontiguousarray(packed.desc)
    with torch.cuda.device(dev):
        check(lib.yb_resize_batch(ptr(packed.pixels), packed.pixels.numel(), desc.ctypes.data_as(C.c_void_p),
                                  ptr(packed.desc_dev), n, new_h, new_w, int(bool(letterbox)), int(interp), ptr(out),
                                  ptr(params), stream_handle()), "yb_resize_batch")
    return out, params


def _resize_packed_interp(packed, new_width, new_height, letterbox, interp, out=None):
    """yb_resize_batch_interp: one OpenCV interpolation (0..4) per image, the tap tables built on the host and sent
    in one pinned H2D copy."""
    n, dev = packed.n, packed.device
    new_w, new_h = int(new_width), int(new_height)
    it = np.asarray(interp, np.int64).reshape(-1)
    if it.size == 1:
        it = np.full(n, int(it[0]), np.int64)
    if it.size != n:
        raise ValueError(f"resize_train_batch: {it.size} interpolations for {n} images")
    if ((it < 0) | (it > 4)).any():
        i = int(np.argmax((it < 0) | (it > 4)))
        raise ValueError(f"resize_train_batch: image {i}: interp must be in 0..4 (cv2.INTER_NEAREST .. INTER_LANCZOS4), "
                         f"got {int(it[i])}")
    it = np.ascontiguousarray(it, np.int32)
    if out is None:
        out = torch.empty((n, new_h, new_w, 3), dtype=torch.float32, device=dev)
    elif (out.dtype != torch.float32 or tuple(out.shape) != (n, new_h, new_w, 3) or not out.is_contiguous()
          or out.device != dev):
        raise ValueError(f"out must be a contiguous float32 [{n}, {new_h}, {new_w}, 3] tensor on {dev}")
    params = torch.empty((n, 4), dtype=torch.float64, device=dev)
    desc = np.ascontiguousarray(packed.desc)
    dp, ip, lb = desc.ctypes.data_as(C.c_void_p), it.ctypes.data_as(C.c_void_p), int(bool(letterbox))
    nbytes = C.c_size_t()
    check(lib.yb_resize_tables_bytes(dp, n, new_h, new_w, lb, ip, C.byref(nbytes)), "yb_resize_tables_bytes")
    host = torch.empty((nbytes.value,), dtype=torch.uint8, pin_memory=True)
    check(lib.yb_resize_tables(dp, n, new_h, new_w, lb, ip, C.c_void_p(host.data_ptr()), nbytes.value),
          "yb_resize_tables")
    with torch.cuda.device(dev):
        tabs = host.to(dev, non_blocking=True)                # the one host -> device copy
        check(lib.yb_resize_batch_interp(ptr(packed.pixels), packed.pixels.numel(), dp, ptr(packed.desc_dev), n, new_h,
                                         new_w, lb, ip, C.c_void_p(host.data_ptr()), ptr(tabs), nbytes.value, ptr(out),
                                         ptr(params), stream_handle()), "yb_resize_batch_interp")
    return out, params


def resize_train_batch(images, new_width, new_height, interp, letterbox=True, out=None, device=None):
    """The resize of parse_data(mode='train') (utils/data_utils.py:160-161) for a batch: resize_with_bbox with each
    image's drawn interpolation, fused with BGR->RGB + float32 / 255.
      images: a PackedImages (augment_train_batch's or decode_jpeg_batch's output: no upload) or a list of uint8 BGR
      [H, W, 3] images; interp: one int or one per image (augment_train_batch's int64 [n]), 0 INTER_NEAREST,
      1 INTER_LINEAR, 2 INTER_CUBIC, 3 INTER_AREA, 4 INTER_LANCZOS4.
    -> (x float32 [n, new_height, new_width, 3] RGB in [0, 1], params float64 [n, 4]) on the device, as
    preprocess_batch returns them, so flip_batch, yb_resize_boxes and process_box_batch follow unchanged.
    Equal to cv2.resize of OpenCV 4.13 byte for byte; for INTER_CUBIC that is OpenCV's own code
    (cv2.ipp.setUseIPP(False)), within 1 of a default cv2 build, which sends it through Intel IPP.  Interp 0 / 1
    images equal preprocess_batch's.  The per-image tap tables are built on the host (yb_resize_tables) and cross
    in one H2D copy; one launch, no host synchronisation."""
    packed = images if isinstance(images, PackedImages) else PackedImages(images, device)
    return _resize_packed_interp(packed, new_width, new_height, letterbox, interp, out)


def preprocess_batch(images, new_width, new_height, letterbox=True, interp=1, out=None, device=None):
    """images: list of uint8 [H, W, 3] BGR images of any sizes (numpy arrays or tensors), or a PackedImages (from
    decode_jpeg_batch: no second upload) ->
    (x float32 [n, new_height, new_width, 3] RGB in [0, 1] on the device, params float64 [n, 4] on the device).

    letterbox=True is letterbox_resize (utils/data_aug.py:274-293, 128-grey border), False a plain stretch to the
    target (cv2.resize(img, (new_width, new_height)), eval.py / test_single_image.py); interp 0 is nearest, 1 OpenCV's
    bilinear (the reference's evaluation inputs, utils/data_utils.py:172).  Then cvtColor(BGR2RGB) + float32 / 255.
    params rows are (resize_ratio, dw, dh, 1) for letterbox, (ori_w / new_w, ori_h / new_h, 0, 0) for stretch: what
    restore_boxes needs.  The images are packed into one pinned buffer, copied with one H2D copy and resized in one
    launch; no host synchronisation."""
    packed = images if isinstance(images, PackedImages) else PackedImages(images, device)
    return _resize_packed(packed, new_width, new_height, letterbox, interp, out)


def resize_with_bbox(img, bbox, new_width, new_height, interp=0, letterbox=False):
    """utils/data_aug.py:296-318 for one image, the reference's signature, with the caller's cvtColor(BGR2RGB) +
    float32 / 255 fused in: -> (x float32 [new_height, new_width, 3] RGB in [0, 1], bbox float32 [V, >=4] transformed
    like the reference), both on the device.  Columns past the fourth (a mix-up weight) are carried unchanged.
    interp 0 / 1 take preprocess_batch's path, 2..4 (cubic, area, Lanczos4) resize_train_batch's."""
    packed = PackedImages([img])
    if interp in (0, 1):
        x, _ = _resize_packed(packed, new_width, new_height, letterbox, interp)
    else:
        x, _ = _resize_packed_interp(packed, new_width, new_height, letterbox, interp)
    a = np.asarray(bbox, np.float32)
    if a.ndim != 2 or a.shape[1] < 4:
        raise ValueError(f"bbox must be [V, >=4], got {a.shape}")
    b = torch.from_numpy(np.ascontiguousarray(a)).to(packed.device)
    if b.shape[0]:
        cnt = torch.tensor([b.shape[0]], dtype=torch.int32, device=packed.device)
        with torch.cuda.device(packed.device):
            check(lib.yb_resize_boxes(ptr(b), ptr(cnt), 1, int(b.shape[0]), int(b.shape[1]), ptr(packed.desc_dev),
                                      int(new_height), int(new_width), int(bool(letterbox)), stream_handle()),
                  "yb_resize_boxes")
    return x[0], b


def restore_boxes(out_boxes, counts, params, inplace=False):
    """test_single_image.py:64-70 for a batch: detections in network-input coordinates (detect_raw's out_boxes
    [n, slots, 4] float32 and counts [n] int32, on the device) -> source-image coordinates, with the params of
    preprocess_batch.  Slots past counts[i] are left as they are.  Returns a new tensor unless inplace."""
    b = out_boxes if inplace else out_boxes.clone()
    if (b.dtype != torch.float32 or b.dim() != 3 or b.shape[2] != 4 or not b.is_contiguous() or not b.is_cuda
            or counts.dtype != torch.int32 or tuple(counts.shape) != (b.shape[0],)
            or params.dtype != torch.float64 or tuple(params.shape) != (b.shape[0], 4)):
        raise ValueError("restore_boxes expects out_boxes float32 [n, slots, 4], counts int32 [n], params float64 [n, 4]")
    if b.shape[1]:
        with torch.cuda.device(b.device):
            check(lib.yb_restore_boxes(ptr(b), ptr(counts.contiguous()), int(b.shape[0]), int(b.shape[1]), 4,
                                       ptr(params.contiguous()), stream_handle()), "yb_restore_boxes")
    return b


def _jpeg_bytes(src):
    if isinstance(src, (bytes, bytearray, memoryview)):
        return bytes(src)
    if isinstance(src, np.ndarray):
        return src.tobytes()
    with open(src, "rb") as f:
        return f.read()


def decode_jpeg_batch(sources, device=None, check=True):
    """cv2.imread (IMREAD_COLOR, EXIF orientation applied) for a batch of baseline JPEG files, on the device:
    sources are bytes-like objects or file paths -> PackedImages of uint8 BGR images equal to cv2.imread's, which
    preprocess_batch / val_batch take without a second upload.

    Headers are parsed on the host first: an unsupported or malformed file raises ValueError naming its index and
    the reason before any device work.  Then one pinned blob (tables + compressed bytes) crosses PCIe and six launches
    decode the whole batch.  Corrupt entropy-coded data gives the image a nonzero status (include/yolob200.h:
    YB_JPEG_*) where libjpeg would warn and fill grey; other images are unaffected.  check=True reads the statuses
    back once (a host synchronisation) and raises ValueError listing the corrupt images; check=False does not
    synchronise, and `packed.status` (int32 [n] on the device) holds the codes."""
    dev = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
    files = [_jpeg_bytes(s) for s in sources]
    n = len(files)
    if n == 0:
        raise ValueError("no images")
    bufs = [C.create_string_buffer(f, len(f)) for f in files]
    ptrs = (C.c_void_p * n)(*[C.cast(b, C.c_void_p) for b in bufs])
    sizes = (C.c_size_t * n)(*[len(f) for f in files])
    blob_bytes = C.c_size_t()
    check_rc(lib.yb_jpeg_pack_bytes(ptrs, sizes, n, C.byref(blob_bytes)), "decode_jpeg_batch")
    host = torch.empty((blob_bytes.value,), dtype=torch.uint8, pin_memory=True)
    desc = np.zeros((n, 4), np.int64)
    check_rc(lib.yb_jpeg_pack(ptrs, sizes, n, C.c_void_p(host.data_ptr()), blob_bytes.value,
                              desc.ctypes.data_as(C.c_void_p)), "decode_jpeg_batch")
    ws_bytes, pix_bytes = C.c_size_t(), C.c_size_t()
    check_rc(lib.yb_jpeg_workspace_bytes(C.c_void_p(host.data_ptr()), n, C.byref(ws_bytes), C.byref(pix_bytes)),
             "decode_jpeg_batch")
    with torch.cuda.device(dev):
        blob = host.to(dev, non_blocking=True)                 # the one host -> device copy
        ws = torch.empty((ws_bytes.value,), dtype=torch.uint8, device=dev)
        data = torch.empty((n * 32 + max(pix_bytes.value, 1),), dtype=torch.uint8, device=dev)
        status = torch.empty((n,), dtype=torch.int32, device=dev)
        check_rc(lib.yb_jpeg_decode(ptr(blob), C.c_void_p(host.data_ptr()), n, ptr(data[n * 32:]), ptr(data),
                                    ptr(status), ptr(ws), ws_bytes.value, stream_handle()), "yb_jpeg_decode")
    packed = PackedImages.from_device(data, desc, status, h2d_bytes=blob_bytes.value)
    if check:
        bad = [(i, int(v)) for i, v in enumerate(status.cpu().tolist()) if v]
        if bad:
            raise ValueError("corrupt JPEG data: " + ", ".join(f"image {i}: {jpeg_status_text(v)}" for i, v in bad))
    return packed


def jpeg_status_text(code):
    names = {_lib.YB_JPEG_BAD_MARKER: "unexpected marker", _lib.YB_JPEG_BAD_RST: "restart markers out of sequence",
             _lib.YB_JPEG_BAD_CODE: "bad Huffman code", _lib.YB_JPEG_BAD_INDEX: "coefficient index past 63",
             _lib.YB_JPEG_TRUNCATED: "data ends before the last MCU"}
    return ", ".join(v for k, v in names.items() if code & k) or "ok"


def jpeg_info(source):
    """yb_jpeg_parse of one file: dict of the oriented height / width, stored size, components, luma sampling,
    restart interval, orientation and mode (0 SOF0, 1 SOF1).  ValueError with the reason when it is not supported."""
    f = _jpeg_bytes(source)
    info = _lib.JpegInfo()
    check_rc(lib.yb_jpeg_parse(f, len(f), C.byref(info)), "jpeg_info")
    return {k: getattr(info, k) for k, _ in info._fields_}


def check_rc(rc, what):
    """check() for the JPEG entry points: an unsupported file is a ValueError as well."""
    if rc == -3:
        raise ValueError(f"{what}: {lib.yb_last_error_string().decode('utf-8', 'replace')}")
    check(rc, what)


def _per_image(name, value, n):
    vals = list(value) if isinstance(value, (list, tuple)) else [value] * n
    if len(vals) != n:
        raise ValueError(f"{name}: {len(vals)} values for {n} images")
    return vals


def encode_jpeg_batch(images, quality=95, sampling="420", restart_interval=0, luma_quality=None, chroma_quality=None,
                      to_host=True, optimize=False, progressive=False, device=None):
    """cv2.imencode('.jpg', img, params) for a batch, on the device: baseline JPEG files equal to OpenCV 4.13's byte
    for byte.  images: a PackedImages (decode_jpeg_batch's output: no upload), or a list of uint8 BGR [H, W, 3] or
    grey [H, W] / [H, W, 1] images as numpy arrays or tensors (CUDA tensors are read in place; host images cross in
    one pinned H2D copy).  Grey gives a one-component file.

    quality, sampling ("411", "420", "422", "440", "444"), restart_interval, luma_quality and chroma_quality are
    IMWRITE_JPEG_QUALITY, _SAMPLING_FACTOR, _RST_INTERVAL, _LUMA_QUALITY and _CHROMA_QUALITY (None: not given), each
    a value for the batch or a list with one per image.  Progressive and optimised-Huffman files are not supported.

    to_host=True returns a list of bytes; reading the lengths is the one synchronisation, then one D2H copy.
    to_host=False returns (data, desc) without synchronising: data a uint8 CUDA tensor with the files back to back
    from offset 0 (its size is an upper bound), desc an int64 [n, 2] CUDA tensor of (offset, length)."""
    if optimize:
        raise ValueError("encode_jpeg_batch: optimised Huffman tables (IMWRITE_JPEG_OPTIMIZE) are not supported")
    if progressive:
        raise ValueError("encode_jpeg_batch: progressive JPEG (IMWRITE_JPEG_PROGRESSIVE) is not supported")
    keep = []                                        # tensors the launches read
    if isinstance(images, PackedImages):
        n, dev = images.n, images.device
        base = images.pixels.data_ptr()
        keep.append(images.data)
        srcs = [(base + int(o), int(h), int(w), 3, int(p)) for o, h, w, p in images.desc.tolist()]
    else:
        images = list(images)
        n = len(images)
        srcs, host = [None] * n, []
        for i, im in enumerate(images):
            t = im if isinstance(im, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(np.asarray(im)))
            if t.dtype != torch.uint8 or t.dim() not in (2, 3) or (t.dim() == 3 and t.shape[2] not in (1, 3)):
                raise ValueError(f"image {i}: expected uint8 [H, W, 3] BGR or [H, W] / [H, W, 1] grey, got "
                                 f"{t.dtype} {tuple(t.shape)}")
            h, w = int(t.shape[0]), int(t.shape[1])
            c = 1 if t.dim() == 2 else int(t.shape[2])
            if not (1 <= h <= 65535 and 1 <= w <= 65535):
                raise ValueError(f"image {i}: size {h} x {w} is outside 1..65535")
            if t.is_cuda:
                t = t.contiguous()
                keep.append(t)
                srcs[i] = (t.data_ptr(), h, w, c, w * c)
            else:
                host.append((i, t.contiguous(), h, w, c))
        if n == 0:
            raise ValueError("encode_jpeg_batch: no images")
        on_dev = [t.device for t in keep]
        dev = torch.device(device if device is not None else
                           on_dev[0] if on_dev else f"cuda:{torch.cuda.current_device()}")
        if host:
            offs, total = [], 0
            for _, t, *_ in host:
                offs.append(total)
                total += (t.numel() + 15) // 16 * 16
            pinned = torch.empty((total,), dtype=torch.uint8, pin_memory=True)
            for o, (_, t, *_) in zip(offs, host):
                pinned[o: o + t.numel()] = t.reshape(-1)
            with torch.cuda.device(dev):
                up = pinned.to(dev, non_blocking=True)           # the one host -> device copy of the pixels
            keep.append(up)
            for o, (i, _, h, w, c) in zip(offs, host):
                srcs[i] = (up.data_ptr() + o, h, w, c, w * c)
    q = _per_image("quality", quality, n)
    sm = _per_image("sampling", sampling, n)
    ri = _per_image("restart_interval", restart_interval, n)
    lq = _per_image("luma_quality", luma_quality, n)
    cq = _per_image("chroma_quality", chroma_quality, n)
    desc = (_lib.JpegEncImage * n)()
    for i, (ptr_i, h, w, c, pitch) in enumerate(srcs):
        if str(sm[i]) not in _lib.YB_JPEG_SAMPLING:
            raise ValueError(f"image {i}: sampling must be one of {sorted(_lib.YB_JPEG_SAMPLING)}, got {sm[i]!r}")
        desc[i] = _lib.JpegEncImage(ptr_i, pitch, h, w, c, int(q[i]), -1 if lq[i] is None else int(lq[i]),
                                    -1 if cq[i] is None else int(cq[i]), _lib.YB_JPEG_SAMPLING[str(sm[i])], int(ri[i]))
    blob_bytes = C.c_size_t()
    check(lib.yb_jpeg_enc_pack_bytes(desc, n, C.byref(blob_bytes)), "encode_jpeg_batch")
    hblob = torch.empty((blob_bytes.value,), dtype=torch.uint8, pin_memory=True)
    check(lib.yb_jpeg_enc_pack(desc, n, C.c_void_p(hblob.data_ptr()), blob_bytes.value), "encode_jpeg_batch")
    ws_bytes, out_bytes = C.c_size_t(), C.c_size_t()
    check(lib.yb_jpeg_enc_workspace_bytes(C.c_void_p(hblob.data_ptr()), n, C.byref(ws_bytes), C.byref(out_bytes)),
          "encode_jpeg_batch")
    with torch.cuda.device(dev):
        blob = hblob.to(dev, non_blocking=True)
        ws = torch.empty((ws_bytes.value,), dtype=torch.uint8, device=dev)
        data = torch.empty((out_bytes.value,), dtype=torch.uint8, device=dev)
        out_desc = torch.empty((n, 2), dtype=torch.int64, device=dev)
        check(lib.yb_jpeg_enc_encode(ptr(blob), C.c_void_p(hblob.data_ptr()), n, ptr(data), out_bytes.value,
                                     ptr(out_desc), ptr(ws), ws_bytes.value, stream_handle()), "yb_jpeg_enc_encode")
    if not to_host:
        return data, out_desc
    d = out_desc.cpu().numpy()                        # the one synchronisation
    total = int(d[-1, 0] + d[-1, 1])
    host = torch.empty((total,), dtype=torch.uint8, pin_memory=True)
    host.copy_(data[:total])                          # the one D2H copy
    buf = host.numpy().tobytes()
    return [buf[o: o + ln] for o, ln in d.tolist()]


def write_jpeg_batch(paths, images, **kw):
    """cv2.imwrite(path, img, params) for a batch: encode_jpeg_batch(images, **kw) written to paths."""
    paths = list(paths)
    files = encode_jpeg_batch(images, **kw)
    if len(paths) != len(files):
        raise ValueError(f"write_jpeg_batch: {len(paths)} paths for {len(files)} images")
    for p, f in zip(paths, files):
        with open(p, "wb") as fh:
            fh.write(f)


# ---------------------------------------------------------------------------------------------------------------------
# Training augmentation: parse_data(mode='train') (utils/data_utils.py:140-165) around the resize.  The draws are made
# here, on the host, from np.random and random in the reference's order; the pixels are one device launch
# (yb_augment_batch) before the resize and one (yb_flip_batch) after it.
# ---------------------------------------------------------------------------------------------------------------------

def bbox_iou(bbox_a, bbox_b, offset=0):
    """IoU matrix [N, M] of boxes (x_min, y_min, x_max, y_max, ...) [N, >=4] and [M, >=4]; `offset` is added to each
    width and height (utils/data_aug.py:93-120)."""
    if bbox_a.shape[1] < 4 or bbox_b.shape[1] < 4:
        raise IndexError("Bounding boxes axis 1 must have at least length 4")
    lo = np.maximum(bbox_a[:, None, :2], bbox_b[None, :, :2])
    hi = np.minimum(bbox_a[:, None, 2:4], bbox_b[None, :, 2:4])
    inter = np.prod(hi - lo + offset, axis=2) * (lo < hi).all(axis=2)
    area_a = np.prod(bbox_a[:, 2:4] - bbox_a[:, :2] + offset, axis=1)
    area_b = np.prod(bbox_b[:, 2:4] - bbox_b[:, :2] + offset, axis=1)
    return inter / (area_a[:, None] + area_b[None, :] - inter)


def bbox_crop(bbox, crop_box=None, allow_outside_center=True):
    """Boxes [N, >=4] clipped to crop_box = (x, y, w, h) (None or 0 entries: unbounded) and shifted to its origin;
    boxes left empty, and unless allow_outside_center those whose centre lies outside, are dropped.  Extra columns
    are carried (utils/data_aug.py:39-91)."""
    out = bbox.copy()
    if crop_box is None:
        return out
    if len(crop_box) != 4:
        raise ValueError(f"Invalid crop_box parameter, requires length 4, given {crop_box}")
    if all(c is None for c in crop_box):
        return out
    x, y, w, h = crop_box
    x, y = (x or 0), (y or 0)
    win = np.array((x, y, x + (w if w else np.inf), y + (h if h else np.inf)))
    keep = np.ones(len(out), bool)
    if not allow_outside_center:
        centre = (out[:, :2] + out[:, 2:4]) / 2
        keep = ((win[:2] <= centre) & (centre < win[2:])).all(axis=1)
    out[:, :2] = np.maximum(out[:, :2], win[:2])
    out[:, 2:4] = np.minimum(out[:, 2:4], win[2:4])
    out[:, :2] -= win[:2]
    out[:, 2:4] -= win[:2]
    keep &= (out[:, :2] < out[:, 2:4]).all(axis=1)
    return out[keep]


_SSD_CONSTRAINTS = ((0.1, None), (0.3, None), (0.5, None), (0.7, None), (0.9, None), (None, 1))


def random_crop_with_constraints(bbox, size, min_scale=0.3, max_scale=1, max_aspect_ratio=2, constraints=None,
                                 max_trial=50):
    """SSD's constrained random crop (utils/data_aug.py:123-217): size = (w, h) -> (boxes, (x, y, w, h)).
    Up to max_trial windows per (min_iou, max_iou) constraint are drawn with `random`; the first one whose IoU with
    every box lies in range joins the candidates, then np.random picks candidates until one keeps a box centre.
    An image without boxes takes the first window drawn.  A window as tall or wide as the image makes
    random.randrange(0) raise ValueError, as in the reference."""
    w, h = size
    picks = [(0, 0, w, h)]
    for lo, hi in (_SSD_CONSTRAINTS if constraints is None else constraints):
        lo = -np.inf if lo is None else lo
        hi = np.inf if hi is None else hi
        for _ in range(max_trial):
            scale = random.uniform(min_scale, max_scale)
            ar = random.uniform(max(1 / max_aspect_ratio, scale * scale), min(max_aspect_ratio, 1 / (scale * scale)))
            ch = int(h * scale / np.sqrt(ar))
            cw = int(w * scale * np.sqrt(ar))
            cy = random.randrange(h - ch)
            cx = random.randrange(w - cw)
            if len(bbox) == 0:
                return bbox, (cx, cy, cw, ch)
            iou = bbox_iou(bbox, np.array(((cx, cy, cx + cw, cy + ch),)))
            if lo <= iou.min() and iou.max() <= hi:
                picks.append((cx, cy, cw, ch))
                break
    while picks:
        crop = picks.pop(np.random.randint(0, len(picks)))
        kept = bbox_crop(bbox, crop, allow_outside_center=False)
        if kept.size:
            return kept, tuple(crop)
    return bbox, (0, 0, w, h)


def _draw_mix():
    r = np.random.beta(1.5, 1.5)
    return max(0, min(1, r))


def _draw_color(brightness_delta=32, hue_vari=18, sat_vari=0.5, val_vari=0.5):
    """random_color_distort's draws -> (brightness delta, hue delta, saturation and value multipliers); an op whose
    coin does not land above 0.5 gets its identity.  Every coin is drawn, taken or not."""
    bright = int(np.random.uniform(-brightness_delta, brightness_delta)) if np.random.uniform(0, 1) > 0.5 else 0
    amount = {"hue": 0, "sat": 1.0, "val": 1.0}
    draws = {"hue": lambda: int(np.random.randint(-hue_vari, hue_vari)),
             "sat": lambda: 1 + np.random.uniform(-sat_vari, sat_vari),
             "val": lambda: 1 + np.random.uniform(-val_vari, val_vari)}
    for op in (("val", "sat", "hue") if np.random.randint(0, 2) else ("sat", "hue", "val")):
        if np.random.uniform(0, 1) > 0.5:
            amount[op] = draws[op]()
    return bright, amount["hue"], amount["sat"], amount["val"]


def _draw_expand(h, w, max_ratio=4, keep_ratio=True):
    """random_expand's draws -> (canvas h, canvas w, off_y, off_x)."""
    rx = random.uniform(1, max_ratio)
    ry = rx if keep_ratio else random.uniform(1, max_ratio)
    oh, ow = int(h * ry), int(w * rx)
    return oh, ow, random.randint(0, oh - h), random.randint(0, ow - w)


def _augment_param(src1, h, w, src2=-1, r=None, color=None, expand=None, crop=None, fill=0):
    """The yb_augment_param of one output; h, w are the mixed image's size."""
    p = _lib.AugmentParam()
    p.src1, p.src2 = src1, src2
    p.w1, p.w2 = (1.0, 0.0) if r is None else (np.float32(r), np.float32(1.0 - r))
    p.canvas_h, p.canvas_w, p.off_y, p.off_x = expand if expand is not None else (h, w, 0, 0)
    p.crop_x, p.crop_y, p.out_w, p.out_h = crop if crop is not None else (0, 0, p.canvas_w, p.canvas_h)
    p.color = int(color is not None)
    p.brightness, p.hue, p.saturation, p.value = color if color is not None else (0, 0, 1.0, 1.0)
    p.fill = int(fill)
    return p


def _augment_launch(packed, params):
    """One yb_augment_batch over `packed` with the records `params` -> PackedImages of the outputs."""
    n = len(params)
    table = (_lib.AugmentParam * n)(*params)
    off = 0
    for p in table:
        p.out_offset = off
        off += (3 * p.out_h * p.out_w + 15) // 16 * 16
    dev = packed.device
    nbytes = C.sizeof(table)
    host = torch.empty((nbytes,), dtype=torch.uint8, pin_memory=True)
    C.memmove(host.data_ptr(), C.addressof(table), nbytes)
    desc = np.ascontiguousarray(packed.desc)
    with torch.cuda.device(dev):
        pdev = host.to(dev, non_blocking=True)                # the one host -> device copy
        data = torch.empty((n * 32 + max(off, 1),), dtype=torch.uint8, device=dev)
        check(lib.yb_augment_batch(ptr(packed.pixels), packed.pixels.numel(), desc.ctypes.data_as(C.c_void_p),
                                   ptr(packed.desc_dev), packed.n, C.cast(table, C.c_void_p), ptr(pdev), n,
                                   ptr(data[n * 32:]), data.numel() - n * 32, ptr(data), stream_handle()),
              "yb_augment_batch")
    out_desc = np.array([(p.out_offset, p.out_h, p.out_w, 3 * p.out_w) for p in table], np.int64).reshape(n, 4)
    return PackedImages.from_device(data, out_desc, h2d_bytes=nbytes)


def _one(img, device=None):
    packed = img if isinstance(img, PackedImages) else PackedImages([img], device)
    h, w = (int(v) for v in packed.desc[0, 1:3])
    return packed, h, w


def mix_up(img1, img2, bbox1, bbox2):
    """utils/data_aug.py:12-36: img1 * r + img2 * (1 - r) on a canvas of the larger sides, r ~ Beta(1.5, 1.5) ->
    (mixed image uint8 [H, W, 3] on the device, boxes float64 [N1 + N2, 5] with r / 1 - r as the last column)."""
    packed = PackedImages([img1, img2])
    (h1, w1), (h2, w2) = packed.desc[0, 1:3].tolist(), packed.desc[1, 1:3].tolist()
    r = _draw_mix()
    out = _augment_launch(packed, [_augment_param(0, max(h1, h2), max(w1, w2), 1, r)])
    b1 = np.concatenate((bbox1, np.full((bbox1.shape[0], 1), r)), axis=-1)
    b2 = np.concatenate((bbox2, np.full((bbox2.shape[0], 1), 1. - r)), axis=-1)
    return out.image(0), np.concatenate((b1, b2), axis=0)


def random_color_distort(img, brightness_delta=32, hue_vari=18, sat_vari=0.5, val_vari=0.5):
    """utils/data_aug.py:220-271: random brightness, then value / saturation / hue in one of two drawn orders through
    OpenCV's 8-bit HSV -> uint8 BGR [H, W, 3] on the device."""
    packed, h, w = _one(img)
    color = _draw_color(brightness_delta, hue_vari, sat_vari, val_vari)
    return _augment_launch(packed, [_augment_param(0, h, w, color=color)]).image(0)


def random_expand(img, bbox, max_ratio=4, fill=0, keep_ratio=True):
    """utils/data_aug.py:349-380: the image placed at a random offset on a canvas up to max_ratio times larger,
    filled with `fill` -> (uint8 [oh, ow, 3] on the device, bbox shifted in place, as the reference does)."""
    packed, h, w = _one(img)
    ex = _draw_expand(h, w, max_ratio, keep_ratio)
    out = _augment_launch(packed, [_augment_param(0, h, w, expand=ex, fill=fill)]).image(0)
    bbox[:, :2] += (ex[3], ex[2])
    bbox[:, 2:4] += (ex[3], ex[2])
    return out, bbox


def _flip_launch(x, flags, boxes=None, counts=None):
    n, h, w = (int(v) for v in x.shape[:3])
    f = torch.as_tensor(np.asarray(flags, np.int32).reshape(-1)).pin_memory().to(x.device, non_blocking=True) \
        if not isinstance(flags, torch.Tensor) else flags.to(x.device, torch.int32, non_blocking=True).contiguous()
    if f.numel() != n:
        raise ValueError(f"flip_batch: {f.numel()} flags for {n} images")
    vmax, ld = (int(boxes.shape[1]), int(boxes.shape[2])) if boxes is not None else (0, 0)
    with torch.cuda.device(x.device):
        check(lib.yb_flip_batch(ptr(x), n, h, w, x.element_size(), ptr(f), ptr(boxes), ptr(counts), vmax, ld,
                                stream_handle()), "yb_flip_batch")
    return x


def flip_batch(x, flags, boxes=None, counts=None):
    """random_flip's horizontal flip after the resize, for a batch: x float32 [n, H, W, 3] (preprocess_batch's output)
    flipped in place where flags[i] is true; boxes float32 [n, vmax, >=4] on the device (the first counts[i], int32,
    of image i) get x' = W - x with min and max swapped.  flags: host booleans (e.g. augment_train_batch's) or a
    device tensor.  One launch, no host synchronisation.  Returns x."""
    if (not isinstance(x, torch.Tensor) or not x.is_cuda or x.dtype != torch.float32 or x.dim() != 4
            or x.shape[3] != 3 or not x.is_contiguous()):
        raise ValueError("flip_batch expects a contiguous float32 [n, H, W, 3] CUDA tensor")
    if boxes is not None:
        if (counts is None or boxes.dtype != torch.float32 or boxes.dim() != 3 or boxes.shape[0] != x.shape[0]
                or boxes.shape[2] < 4 or not boxes.is_contiguous() or boxes.device != x.device
                or counts.dtype != torch.int32 or tuple(counts.shape) != (x.shape[0],) or counts.device != x.device):
            raise ValueError("flip_batch: boxes must be float32 [n, vmax, >=4] with counts int32 [n], on x's device")
        if boxes.shape[1] == 0:
            boxes = counts = None
    return _flip_launch(x, flags, boxes, counts)


def random_flip(img, bbox, px=0, py=0):
    """utils/data_aug.py:323-346: horizontal flip with probability px, then vertical with py (both coins always
    drawn).  img uint8 or float32 [H, W, 3] (numpy or CUDA tensor) -> (flipped copy on the device, bbox flipped in
    place on the host in its own dtype)."""
    t = torch.from_numpy(np.ascontiguousarray(img)) if isinstance(img, np.ndarray) else img
    if t.dim() != 3 or t.shape[2] != 3 or t.dtype not in (torch.uint8, torch.float32):
        raise ValueError(f"random_flip expects a uint8 or float32 [H, W, 3] image, got {t.dtype} {tuple(t.shape)}")
    height, width = int(t.shape[0]), int(t.shape[1])
    fx = np.random.uniform(0, 1) < px
    fy = np.random.uniform(0, 1) < py
    x = t.to(f"cuda:{torch.cuda.current_device()}" if not t.is_cuda else t.device, copy=True).contiguous()
    if fx or fy:
        _flip_launch(x[None], [int(fx) | 2 * int(fy)])
    if fx:
        bbox[:, 0], bbox[:, 2] = width - bbox[:, 2], width - bbox[:, 0].copy()
    if fy:
        bbox[:, 1], bbox[:, 3] = height - bbox[:, 3], height - bbox[:, 1].copy()
    return x, bbox


def augment_train_batch(images, boxes_list, labels_list, mix_with=None, device=None):
    """parse_data(mode='train') (utils/data_utils.py:118-165) for a batch, up to its resize: for image i, drawing from
    np.random and random exactly as the reference does, in this order: the mix-up weight (when mix_with[i] names
    the partner image j, as get_batch_data's pairing would), the colour coins and amounts, the expand coin and
    expand, every crop trial and pick, the interpolation, and both flip coins.
      images: uint8 BGR [H, W, 3] images or a PackedImages (decode_jpeg_batch's output: no upload); boxes_list: per
      image [V, 4] (x_min, y_min, x_max, y_max); labels_list: per image [V] ints; mix_with: None or, per image,
      None or the index of its partner.
    -> (PackedImages of the cropped uint8 images, boxes, labels, interp int64 [n], flip bool [n]).  boxes[i] is host
    numpy as the reference holds it: float32 [N, 5] with a weight column of 1, float64 after a mix-up.  labels[i] is
    labels[:len(boxes[i])]: the reference drops boxes in the crop but not their labels, and process_box pairs box k
    with label k, so this keeps its pairing.  interp[i] (0..4) is for resize_train_batch; flip[i] is for flip_batch
    after the resize.  Pixels: one H2D copy of the parameter table and one launch, no
    host synchronisation."""
    packed = images if isinstance(images, PackedImages) else PackedImages(images, device)
    n = packed.n
    if len(boxes_list) != n or len(labels_list) != n:
        raise ValueError(f"augment_train_batch: {n} images, {len(boxes_list)} box and {len(labels_list)} label arrays")
    mix_with = [None] * n if mix_with is None else list(mix_with)
    if len(mix_with) != n:
        raise ValueError(f"augment_train_batch: mix_with has {len(mix_with)} entries for {n} images")
    gt = []
    for i, (b, l) in enumerate(zip(boxes_list, labels_list)):
        b = np.asarray(b, np.float32)
        b = b.reshape(0, 4) if b.size == 0 else b
        l = np.asarray(l, np.int64).reshape(-1)
        if b.ndim != 2 or b.shape[1] != 4 or len(b) != len(l):
            raise ValueError(f"augment_train_batch: image {i}: boxes {b.shape} and labels {l.shape} do not pair")
        gt.append((b, l))
    sizes = packed.desc[:, 1:3].tolist()
    params, boxes_out, labels_out = [], [], []
    interp, flip = np.zeros(n, np.int64), np.zeros(n, bool)
    for i in range(n):
        j = mix_with[i]
        b1, l1 = gt[i]
        h, w = sizes[i]
        if j is None:
            r = None
            boxes = np.concatenate((b1, np.ones((len(b1), 1), np.float32)), axis=-1)
            labels = l1
        else:
            j = int(j)
            if not 0 <= j < n:
                raise ValueError(f"augment_train_batch: image {i} is paired with image {j} of {n}")
            b2, l2 = gt[j]
            h, w = max(h, sizes[j][0]), max(w, sizes[j][1])
            r = _draw_mix()
            boxes = np.concatenate((np.concatenate((b1, np.full((len(b1), 1), r)), -1),
                                    np.concatenate((b2, np.full((len(b2), 1), 1. - r)), -1)), 0)
            labels = np.concatenate((l1, l2))
        color = _draw_color()
        ex = None
        if np.random.uniform(0, 1) > 0.5:
            ex = _draw_expand(h, w)
            boxes[:, :2] += (ex[3], ex[2])
            boxes[:, 2:4] += (ex[3], ex[2])
        ch, cw = ex[:2] if ex is not None else (h, w)
        boxes, crop = random_crop_with_constraints(boxes, (cw, ch))
        interp[i] = np.random.randint(0, 5)
        flip[i] = np.random.uniform(0, 1) < 0.5
        np.random.uniform(0, 1)                               # random_flip's vertical coin (py = 0)
        params.append(_augment_param(i, h, w, -1 if j is None else j, r, color, ex, crop))
        boxes_out.append(boxes)
        labels_out.append(labels[:len(boxes)])
    return _augment_launch(packed, params), boxes_out, labels_out, interp, flip
