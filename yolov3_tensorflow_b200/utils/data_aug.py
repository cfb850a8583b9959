"""utils/data_aug.py of the reference, the functions on the inference and evaluation input path: `letterbox_resize`
(:274-293) and `resize_with_bbox` (:296-318), fused with the caller's BGR->RGB + float32 / 255
(test_single_image.py:44-46) into device kernels (libyolob200.so: yb_letterbox_normalize for one image, yb_resize_batch
for a batch of images of different sizes, letterbox or stretch, nearest or bilinear), plus the detections' way back to
the source image (test_single_image.py:64-70, yb_restore_boxes).  Bit-exact vs cv2.resize(..., interpolation=0 / 1) of
OpenCV 4.13; the random augmentations of training are CPU image I/O and out of scope."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

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
    """images: list of uint8 [H, W, 3] BGR images of any sizes (numpy arrays or tensors) ->
    (x float32 [n, new_height, new_width, 3] RGB in [0, 1] on the device, params float64 [n, 4] on the device).

    letterbox=True is letterbox_resize (utils/data_aug.py:274-293, 128-grey border), False a plain stretch to the
    target (cv2.resize(img, (new_width, new_height)), eval.py / test_single_image.py); interp 0 is nearest, 1 OpenCV's
    bilinear (the reference's evaluation inputs, utils/data_utils.py:172).  Then cvtColor(BGR2RGB) + float32 / 255.
    params rows are (resize_ratio, dw, dh, 1) for letterbox, (ori_w / new_w, ori_h / new_h, 0, 0) for stretch: what
    restore_boxes needs.  The images are packed into one pinned buffer, copied with one H2D copy and resized in one
    launch; no host synchronisation."""
    packed = PackedImages(images, device)
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
