"""utils/data_aug.py of the reference, the functions on the inference and evaluation input path: `letterbox_resize`
(:274-293) and `resize_with_bbox` (:296-318), fused with the caller's BGR->RGB + float32 / 255
(test_single_image.py:44-46) into device kernels (libyolob200.so: yb_letterbox_normalize for one image, yb_resize_batch
for a batch of images of different sizes, letterbox or stretch, nearest or bilinear), plus the detections' way back to
the source image (test_single_image.py:64-70, yb_restore_boxes).  Bit-exact vs cv2.resize(..., interpolation=0 / 1) of
OpenCV 4.13; the random augmentations of training are CPU image I/O and out of scope.  `decode_jpeg_batch` replaces
the cv2.imread in front of them (utils/data_utils.py:130, test_single_image.py:38): baseline JPEG files decoded on the
device (yb_jpeg_decode), equal to cv2.imread byte for byte, straight into the PackedImages layout.
`encode_jpeg_batch` / `write_jpeg_batch` are cv2.imencode('.jpg') / cv2.imwrite (test_single_image.py:85) for a batch
on the device (yb_jpeg_enc_encode), byte for byte."""
from __future__ import annotations

import ctypes as C

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
    like the reference), both on the device.  Columns past the fourth (a mix-up weight) are carried unchanged."""
    packed = PackedImages([img])
    x, _ = _resize_packed(packed, new_width, new_height, letterbox, interp)
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
