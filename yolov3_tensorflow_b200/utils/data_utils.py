"""utils/data_utils.py of the reference, the part on the hot path's input side: `process_box` (ground-truth lists ->
y_true_13 / _26 / _52, utils/data_utils.py:51-115) as ONE device call for a whole batch (libyolob200.so: yb_process_box).
The box lists (24 B per box) are what crosses PCIe; the 3.66 MB-per-image tensors are built in HBM, bit-identical to
the reference's numpy loop (list order decides collisions: the last box of a slot wins, class bits accumulate).
`val_batch` is parse_data(mode='val') for a whole batch: images resized from uint8 on the device, boxes transformed
the same way, then process_box_batch."""
from __future__ import annotations

import numpy as np
import torch

from .. import _lib
from .._lib import lib, check, ptr, stream_handle


def pack_gt(boxes_list, labels_list, vmax=None):
    """Per-image (boxes [V,5] float32, labels [V] int) lists -> padded host arrays (boxes [n,vmax,5], labels [n,vmax]
    int32, counts [n] int32) in pinned memory, ready for one H2D copy."""
    n = len(boxes_list)
    if n == 0 or n != len(labels_list):
        raise ValueError("pack_gt: need one label array per box array")
    counts = np.asarray([len(b) for b in boxes_list], np.int32)
    vmax = int(vmax or max(1, counts.max()))
    if counts.max() > vmax:
        raise ValueError(f"pack_gt: {counts.max()} boxes > vmax {vmax}")
    hb = torch.zeros((n, vmax, 5), dtype=torch.float32).pin_memory()
    hl = torch.zeros((n, vmax), dtype=torch.int32).pin_memory()
    for i, (b, l) in enumerate(zip(boxes_list, labels_list)):
        b = np.asarray(b, np.float32).reshape(-1, 5)
        if len(b) != len(l):
            raise ValueError(f"pack_gt: image {i}: {len(b)} boxes but {len(l)} labels")
        hb[i, :len(b)] = torch.from_numpy(b)
        hl[i, :len(b)] = torch.from_numpy(np.asarray(l, np.int64).astype(np.int32))
    return hb, hl, torch.from_numpy(counts).pin_memory()


def process_box_batch(boxes, labels, counts, img_size, class_num, anchors, device=None, out=None):
    """boxes [n,vmax,5] float32 (x_min, y_min, x_max, y_max, mixup weight), labels [n,vmax] int32, counts [n] int32
    (host or CUDA tensors; host tensors are copied asynchronously), img_size = [W, H] like the reference ->
    (y_true_13 [n,H/32,W/32,3,6+C], y_true_26, y_true_52) float32 on the device.  No host synchronisation."""
    dev = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
    b = boxes.to(dev, non_blocking=True).contiguous()
    l = labels.to(dev, non_blocking=True).contiguous()
    c = counts.to(dev, non_blocking=True).contiguous()
    if b.dtype != torch.float32 or l.dtype != torch.int32 or c.dtype != torch.int32:
        raise TypeError("process_box_batch expects float32 boxes and int32 labels / counts")
    n, vmax = int(b.shape[0]), int(b.shape[1])
    if tuple(b.shape) != (n, vmax, 5) or tuple(l.shape) != (n, vmax) or tuple(c.shape) != (n,):
        raise ValueError(f"process_box_batch: shapes {tuple(b.shape)} / {tuple(l.shape)} / {tuple(c.shape)}")
    W, H = int(img_size[0]), int(img_size[1])
    anchors = np.asarray(anchors, np.float32).reshape(9, 2)
    E1 = 6 + int(class_num)
    if out is None:
        out = [torch.empty((n, H // s, W // s, 3, E1), dtype=torch.float32, device=dev) for s in (32, 16, 8)]
    with torch.cuda.device(dev):
        check(lib.yb_process_box(ptr(b), ptr(l), ptr(c), n, vmax, W, H, int(class_num), _lib.fptr(anchors.reshape(-1)),
                                 ptr(out[0]), ptr(out[1]), ptr(out[2]), stream_handle()), "yb_process_box")
    return out[0], out[1], out[2]


def val_batch(images, boxes_list, labels_list, img_size, class_num, anchors, letterbox_resize=True, device=None):
    """parse_data(mode='val') (utils/data_utils.py:166-182) for a batch, on the device: resize_with_bbox(interp=1,
    letterbox=letterbox_resize) + cvtColor(BGR2RGB) + float32 / 255 for the images (one H2D copy of the uint8 pixels,
    one launch), the same box transform, then process_box_batch.
      images: uint8 [H, W, 3] BGR images of any sizes, or a PackedImages (decode_jpeg_batch); boxes_list: per image float32 [V, 4] (x_min, y_min, x_max,
      y_max in source pixels) or [V, 5] with a mix-up weight (1 when absent, as parse_data adds); labels_list: per
      image [V] ints; img_size: [W, H], multiples of 32.
    -> (x [n, H, W, 3], y_true_13, y_true_26, y_true_52), float32 on the device, no host synchronisation."""
    from .data_aug import PackedImages, _resize_packed
    n = len(images)
    if n != len(boxes_list):
        raise ValueError(f"val_batch: {n} images but {len(boxes_list)} box arrays")
    bl = []
    for i, b in enumerate(boxes_list):
        b = np.asarray(b, np.float32)
        b = b.reshape(-1, b.shape[-1] if b.size else 4)
        if b.shape[1] == 4:
            b = np.concatenate([b, np.ones((len(b), 1), np.float32)], 1)
        if b.shape[1] != 5:
            raise ValueError(f"val_batch: image {i}: boxes must be [V, 4] or [V, 5], got {b.shape}")
        bl.append(b)
    W, H = int(img_size[0]), int(img_size[1])
    packed = images if isinstance(images, PackedImages) else PackedImages(images, device)
    dev = packed.device
    x, _ = _resize_packed(packed, W, H, letterbox_resize, 1)
    hb, hl, hc = pack_gt(bl, labels_list)
    b = hb.to(dev, non_blocking=True)
    c = hc.to(dev, non_blocking=True)
    with torch.cuda.device(dev):
        check(lib.yb_resize_boxes(ptr(b), ptr(c), n, int(b.shape[1]), 5, ptr(packed.desc_dev), H, W,
                                  int(bool(letterbox_resize)), stream_handle()), "yb_resize_boxes")
    y13, y26, y52 = process_box_batch(b, hl, c, [W, H], class_num, anchors, device=dev)
    return x, y13, y26, y52


def process_box(boxes, labels, img_size, class_num, anchors):
    """utils/data_utils.py:51-115 for ONE image, the reference's signature: boxes [N,5] float32, labels [N] int64,
    img_size [W, H], anchors [9,2] -> (y_true_13, y_true_26, y_true_52) as CUDA tensors [H/s, W/s, 3, 6+class_num]."""
    hb, hl, hc = pack_gt([np.asarray(boxes, np.float32).reshape(-1, 5)], [np.asarray(labels).reshape(-1)])
    y = process_box_batch(hb, hl, hc, img_size, class_num, anchors)
    return y[0][0], y[1][0], y[2][0]
