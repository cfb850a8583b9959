"""Drawing detections on the device: the reference's utils/plot_utils.py, equal to OpenCV 4.13's pixels bit for bit.

get_color_table is the reference's, on the host.  plot_one_box and plot_detections draw with yb_plot_boxes
(csrc/plot.cu): cv2.rectangle, the filled label box and cv2.putText(FONT_HERSHEY_SIMPLEX, LINE_AA) per detection,
in order, at every line thickness 0..1023.
"""
import ctypes as C
import random

import numpy as np
import torch

from .. import _lib
from .._lib import check, lib, ptr, stream_handle
from .data_aug import PackedImages


def get_color_table(class_num, seed=2):
    """The reference's colour table: reseeds the global random module, three randint(0, 255) per class."""
    random.seed(seed)
    color_table = {}
    for i in range(class_num):
        color_table[i] = [random.randint(0, 255) for _ in range(3)]
    return color_table


def line_thickness_for(h, w, line_thickness=None):
    """plot_one_box's tl: line_thickness, else int(round(0.002 * max(h, w))) (0 up to 250 pixels)."""
    return line_thickness or int(round(0.002 * max(h, w)))


def label_layout(name, tl, c1, score=None):
    """yb_plot_label_layout: the label plot_one_box draws at corner c1 = (x, y) for line thickness tl, name followed
    by ', {:.2f}%' of the float32 score * 100 when score is given.  Returns dict(text, thickness, t_size, c2, org)."""
    raw = name.encode("utf-8") if isinstance(name, str) else bytes(name)
    text = (C.c_uint8 * (len(raw) + _lib.YB_PLOT_SUFFIX_MAX))()
    L = _lib.PlotLayout()
    s = float(np.float32(0 if score is None else score))
    check(lib.yb_plot_label_layout(raw, len(raw), score is not None, s, int(tl), int(c1[0]), int(c1[1]), text,
                                   C.byref(L)), "yb_plot_label_layout")
    return dict(text=bytes(text[:L.length]).decode("ascii"), thickness=L.thickness, t_size=(L.text_w, L.text_h),
                c2=(L.rect_x1, L.rect_y1), org=(L.org_x, L.org_y))


def _draw(packed, boxes, scores, labels, counts, names, colors, tls, with_score, check_status):
    """One yb_plot_boxes launch over a PackedImages.  names: bytes per class (None: no label), colors: 3 ints per
    class, tls: line thickness per image."""
    n, dev = packed.n, packed.device
    classes = len(names)
    blob_names = b"".join(x for x in names if x)
    name_len = (C.c_int * classes)(*[-1 if x is None else len(x) for x in names])
    nbytes = C.c_size_t()
    check(lib.yb_plot_workspace_bytes(n, classes, len(blob_names), C.byref(nbytes)), "yb_plot_workspace_bytes")
    host = torch.empty((nbytes.value,), dtype=torch.uint8, pin_memory=True)
    tl_arr = (C.c_int * n)(*[int(t) for t in tls])
    col_arr = (C.c_int * (3 * classes))(*[int(v) for c in colors for v in c])
    check(lib.yb_plot_pack(tl_arr, n, col_arr, blob_names, name_len, classes, int(with_score),
                           C.c_void_p(host.data_ptr()), nbytes.value), "yb_plot_pack")

    def dev_t(x, dtype, shape):
        t = torch.as_tensor(x).to(device=dev, dtype=dtype).contiguous()
        if tuple(t.shape) != shape:
            raise ValueError(f"plot_detections: expected shape {shape}, got {tuple(t.shape)}")
        return t
    counts = dev_t(counts, torch.int32, (n,))
    slots = int(torch.as_tensor(boxes).shape[1]) if torch.as_tensor(boxes).dim() == 3 else -1
    boxes = dev_t(boxes, torch.float32, (n, slots, 4))
    labels = dev_t(labels, torch.int32, (n, slots))
    scores = dev_t(scores, torch.float32, (n, slots)) if with_score else None
    with torch.cuda.device(dev):
        blob = host.to(dev, non_blocking=True)
        status = torch.empty((n, 2), dtype=torch.int32, device=dev)
        check(lib.yb_plot_boxes(ptr(packed.data), n, int(packed.desc[:, 1].max()), int(packed.desc[:, 2].max()),
                                ptr(boxes), ptr(scores), ptr(labels), ptr(counts), slots, ptr(blob), ptr(status),
                                stream_handle()), "yb_plot_boxes")
    packed.plot_status = status
    if check_status:
        for i, (flags, slot) in enumerate(status.cpu().tolist()):
            if flags:
                what = " and ".join(w for f, w in ((_lib.YB_PLOT_BAD_LABEL, f"a label outside [0, {classes})"),
                                                   (_lib.YB_PLOT_BAD_BOX, "a non-finite coordinate")) if flags & f)
                raise ValueError(f"plot_detections: image {i}: detection {slot} (first of its kind) has {what}; "
                                 "such detections are skipped")
    return status


def plot_detections(images, boxes, scores, labels, counts, class_names, color_table=None, line_thickness=None,
                    check=True):
    """test_single_image.py:81-83 for a batch: for each image i and detection j < counts[i], in order,
    plot_one_box(img_i, boxes[i, j], label=class_names[labels[i, j]] + ', {:.2f}%'.format(scores[i, j] * 100),
    color=color_table[labels[i, j]], line_thickness=line_thickness).

    images: a PackedImages (decode_jpeg_batch's output, drawn in place), or a list of uint8 BGR [H, W, 3] images
    (numpy arrays or tensors, packed once).  boxes [n, slots, 4] float32 in image coordinates (restore_boxes'
    output), scores [n, slots] float32, labels [n, slots] int32, counts [n] int32, preferably on the device.
    color_table: {class: [b, g, r]} or a list; None takes get_color_table(len(class_names)), as the reference does.

    A detection with a label outside [0, len(class_names)) or a non-finite coordinate is skipped and recorded in
    the returned batch's plot_status (int32 [n, 2]: YB_PLOT_* flags, first such slot).  check=True reads it (one
    synchronisation) and raises ValueError naming the image and slot; check=False does not synchronise.
    Returns the PackedImages, ready for encode_jpeg_batch."""
    packed = images if isinstance(images, PackedImages) else PackedImages(list(images))
    if color_table is None:
        color_table = get_color_table(len(class_names))
    colors = [list(color_table[c]) for c in range(len(class_names))]
    tls = [line_thickness_for(int(h), int(w), line_thickness) for _, h, w, _ in packed.desc.tolist()]
    names = [str(nm).encode("utf-8") for nm in class_names]
    _draw(packed, boxes, scores, labels, counts, names, colors, tls, True, check)
    return packed


def _clamped_int(v):
    return max(-(1 << 24), min(1 << 24, int(v)))


def plot_one_box(img, coord, label=None, color=None, line_thickness=None):
    """The reference's plot_one_box, drawn in place on the device.  img: a uint8 [H, W, 3] CUDA tensor with unit
    channel stride and pixel stride 3 (such as PackedImages.image(i)), or a numpy array (one upload, one download).
    coord: [x_min, y_min, x_max, y_max]; color None draws the reference's random.randint colour."""
    tl = line_thickness or int(round(0.002 * max(img.shape[0:2])))
    color = color or [random.randint(0, 255) for _ in range(3)]
    c = [_clamped_int(v) for v in coord[:4]]                # int() as the reference truncates, on the host
    box = torch.tensor([[c]], dtype=torch.float32)
    name = [label.encode("utf-8") if label else None]
    if isinstance(img, torch.Tensor):
        if (img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3 or not img.is_cuda
                or img.stride(2) != 1 or img.stride(1) != 3):
            raise ValueError("plot_one_box: expected a uint8 [H, W, 3] CUDA tensor with pixel stride 3 or a numpy array")
        h, w = int(img.shape[0]), int(img.shape[1])
        desc = torch.zeros((1, 4), dtype=torch.int64)
        data = torch.empty((32,), dtype=torch.uint8, device=img.device)
        desc[0] = torch.tensor([img.data_ptr() - data.data_ptr() - 32, h, w, img.stride(0)])
        data.copy_(desc.view(torch.uint8).reshape(-1))
        packed = PackedImages.from_device(data, desc.numpy())
        _draw(packed, box, None, torch.zeros((1, 1), dtype=torch.int32), torch.ones(1, dtype=torch.int32), name,
              [color], [tl], False, False)
        return img
    a = np.asarray(img)
    packed = PackedImages([a])
    _draw(packed, box, None, torch.zeros((1, 1), dtype=torch.int32), torch.ones(1, dtype=torch.int32), name,
          [color], [tl], False, False)
    img[...] = packed.image(0).cpu().numpy()
    return img
