"""CPU ORACLE — TEST INFRASTRUCTURE ONLY.  Never imported by the product package.

A CPU restatement (numpy fp32 + torch-CPU conv2d) of the YOLOv3 hot path of
wizyoung/YOLOv3_TensorFlow.  Only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import this file.

PARITY PINNING STATUS
  * Everything the reference writes in *Python* (layer wiring, decode, loss
    algebra, gpu_nms filtering/concat, process_box) is pinned: the generator
    ``tests/golden/make_golden.py`` executes the reference's own ``model.py`` /
    ``utils/*.py`` sources over a numpy-backed ``tensorflow`` shim and the golden
    vectors it writes are checked against this file (tests/test_oracle_golden.py).
  * The TensorFlow *kernels* underneath (conv2d, fused batch-norm,
    non_max_suppression, sigmoid_cross_entropy_with_logits, autodiff) are an
    un-vendored third-party dependency (``tensorflow >= 1.8.0`` unpinned,
    the reference's README.md:24) that cannot be installed here (Python 3.12, no
    network): for those this oracle restates TF's published semantics
    (SURVEY.md Appendix B) and is **parity unpinned**.

Every function cites the reference file:line it follows (paths relative to
the reference checkout).
"""
from __future__ import annotations

import math
import numpy as np
import torch
import torch.nn.functional as F

F32 = np.float32

COCO_ANCHORS = np.array(
    [[10, 13], [16, 30], [33, 23], [30, 61], [62, 45], [59, 119], [116, 90], [156, 198], [373, 326]],
    dtype=np.float32,
)  # data/yolo_anchors.txt


# --------------------------------------------------------------------------------------
# Architecture walk (utils/layer_utils.py:24-79, model.py:50-78)
# --------------------------------------------------------------------------------------
def conv_specs(class_num: int = 80, with_div: bool = False):
    """Creation-order list of (scope, cin, cout, k, stride, has_bn) for the 75 convs
    (+ the input down-sampling factor when with_div).

    Written as the same nested walk as the reference (darknet53_body/res_block/
    yolo_block), *not* as a flat table, so it is independent of the product's table.
    """
    specs = []
    state = {"c": 3, "div": 1}

    def conv(scope, filters, k, s=1, bn=True):  # utils/layer_utils.py:9-22
        specs.append((scope, state["c"], filters, k, s, bn) + ((state["div"],) if with_div else ()))
        state["c"] = filters
        state["div"] *= s

    def res_block(filters):  # utils/layer_utils.py:25-32
        conv("darknet53_body", filters, 1)
        conv("darknet53_body", filters * 2, 3)

    # utils/layer_utils.py:35-66
    conv("darknet53_body", 32, 3, 1)
    conv("darknet53_body", 64, 3, 2)
    res_block(32)
    conv("darknet53_body", 128, 3, 2)
    for _ in range(2):
        res_block(64)
    conv("darknet53_body", 256, 3, 2)
    for _ in range(8):
        res_block(128)
    conv("darknet53_body", 512, 3, 2)
    for _ in range(8):
        res_block(256)
    conv("darknet53_body", 1024, 3, 2)
    for _ in range(4):
        res_block(512)

    def yolo_block(cin, filters):  # utils/layer_utils.py:71-79
        state["c"] = cin
        for i in range(3):
            conv("yolov3_head", filters, 1)
            conv("yolov3_head", filters * 2, 3)

    D = 3 * (5 + class_num)
    yolo_block(1024, 512)  # model.py:54
    conv("yolov3_head", D, 1, 1, bn=False)  # model.py:55-57
    state["c"] = 512
    conv("yolov3_head", 256, 1)  # model.py:60
    state["div"] = 16  # upsample (model.py:61)
    yolo_block(256 + 512, 256)  # model.py:62,64
    conv("yolov3_head", D, 1, 1, bn=False)  # model.py:65-67
    state["c"] = 256
    conv("yolov3_head", 128, 1)  # model.py:70
    state["div"] = 8  # upsample (model.py:71)
    yolo_block(128 + 256, 128)  # model.py:72,74
    conv("yolov3_head", D, 1, 1, bn=False)  # model.py:75-77
    return specs


def count_params(class_num: int = 80) -> int:
    """Float count of the darknet .weights payload (SURVEY.md §8c KAT: 62,001,757)."""
    n = 0
    for _, cin, cout, k, _, bn in conv_specs(class_num):
        n += k * k * cin * cout + (4 * cout if bn else cout)
    return n


def forward_flops(h: int, w: int, class_num: int = 80) -> int:
    """2*MAC of the 75 convs per image (SURVEY.md §8c KAT: 65.864 GFLOP @416)."""
    fl = 0
    for _, cin, cout, k, s, bn, div in conv_specs(class_num, with_div=True):
        fl += 2 * (h // (div * s)) * (w // (div * s)) * cout * cin * k * k
    return fl


def make_params(class_num: int = 80, seed: int = 1, det_scale: float = 1.0, conf_bias: float = 0.0,
                random_bn: bool = False):
    """Seeded parameters, one dict per conv in creation order.

    Glorot-uniform conv weights (slim default xavier_initializer), gamma=1, beta=0,
    mean=0, var=1, zero detection bias (model.py:55-57).  ``random_bn`` perturbs the BN
    parameters (tests need non-trivial statistics); ``det_scale``/``conf_bias``
    implement the SURVEY.md §8d config-2 trick so that scores straddle 0.3.
    Weights are HWIO float32 like the TF variables.
    """
    rng = np.random.default_rng(seed)
    params = []
    for scope, cin, cout, k, s, bn in conv_specs(class_num):
        lim = math.sqrt(6.0 / (k * k * cin + k * k * cout))
        w = rng.uniform(-lim, lim, size=(k, k, cin, cout)).astype(F32)
        if bn:
            if random_bn:
                p = dict(
                    w=w,
                    gamma=rng.uniform(0.5, 1.5, cout).astype(F32),
                    beta=rng.uniform(-0.2, 0.2, cout).astype(F32),
                    mean=rng.uniform(-0.1, 0.1, cout).astype(F32),
                    var=rng.uniform(0.5, 1.5, cout).astype(F32),
                )
            else:
                p = dict(w=w, gamma=np.ones(cout, F32), beta=np.zeros(cout, F32),
                         mean=np.zeros(cout, F32), var=np.ones(cout, F32))
        else:
            w = (w * det_scale).astype(F32)
            b = np.zeros(cout, F32)
            if conf_bias != 0.0:
                b.reshape(3, -1)[:, 4] = conf_bias
            p = dict(w=w, b=b)
        params.append(p)
    return params


# --------------------------------------------------------------------------------------
# Forward (model.py:30-80, utils/layer_utils.py) — torch CPU, NHWC in / NHWC out
# --------------------------------------------------------------------------------------
def _round_store(t: torch.Tensor, emulate):
    if emulate is None:
        return t
    dt = torch.float16 if emulate in ("fp16", "float16") else torch.bfloat16
    return t.to(dt).to(t.dtype)


class _Net:
    """Replays the reference graph on torch-CPU tensors (NCHW internally)."""

    def __init__(self, params, is_training, emulate, bn_decay, dtype, record):
        self.p = params
        self.i = 0
        self.training = is_training
        self.emulate = emulate
        self.decay = bn_decay
        self.dtype = dtype
        self.new_stats = []   # (mean, var) moving stats after the UPDATE_OPS (train mode)
        self.record = record  # optional list receiving every conv output (NHWC numpy)

    def _t(self, a):
        return a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a)).to(self.dtype)

    def conv2d(self, x, filters, k, strides=1, bn=True, shortcut=None):
        # utils/layer_utils.py:9-22 : stride 1 -> SAME ; stride 2 -> pad 1 then VALID
        p = self.p[self.i]
        self.i += 1
        w = self._t(p["w"])
        assert w.shape == (k, k, x.shape[1], filters), (w.shape, k, x.shape, filters)
        if self.emulate is not None:
            w = _round_store(w, self.emulate)
        wt = w.permute(3, 2, 0, 1).contiguous()  # HWIO -> OIHW, cross-correlation [TF]
        y = F.conv2d(x, wt, None, stride=strides, padding=k // 2)
        if bn:
            gamma, beta = self._t(p["gamma"]), self._t(p["beta"])
            if self.training:
                # [TF] fused batch norm: batch mean / biased var for normalisation,
                # moving stats updated with the unbiased variance (SURVEY.md B.1)
                mean = y.mean(dim=(0, 2, 3))
                var = y.var(dim=(0, 2, 3), unbiased=False)
                n = y.numel() // y.shape[1]
                d = self.decay
                mm = self._t(p["mean"]) * d + (1 - d) * mean.detach()
                mv = self._t(p["var"]) * d + (1 - d) * var.detach() * (n / max(n - 1, 1))
                self.new_stats.append((mm, mv))
            else:
                mean, var = self._t(p["mean"]), self._t(p["var"])
            scale = gamma / torch.sqrt(var + 1e-5)   # model.py:37 epsilon
            shift = beta - mean * scale
            y = y * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)
            y = torch.where(y > 0, y, 0.1 * y)       # model.py:47 leaky_relu alpha 0.1
        else:
            y = y + self._t(p["b"]).view(1, -1, 1, 1)  # model.py:55-57 bias, linear
        if shortcut is not None:
            y = y + shortcut                          # utils/layer_utils.py:30 add after act
        if bn:
            y = _round_store(y, self.emulate)
        if self.record is not None:
            self.record.append(y.detach().permute(0, 2, 3, 1).contiguous())
        return y

    def res_block(self, x, filters):  # utils/layer_utils.py:25-32
        net = self.conv2d(x, filters, 1)
        return self.conv2d(net, filters * 2, 3, shortcut=x)

    def darknet53_body(self, x):  # utils/layer_utils.py:24-68
        net = self.conv2d(x, 32, 3, 1)
        net = self.conv2d(net, 64, 3, 2)
        net = self.res_block(net, 32)
        net = self.conv2d(net, 128, 3, 2)
        for _ in range(2):
            net = self.res_block(net, 64)
        net = self.conv2d(net, 256, 3, 2)
        for _ in range(8):
            net = self.res_block(net, 128)
        route_1 = net
        net = self.conv2d(net, 512, 3, 2)
        for _ in range(8):
            net = self.res_block(net, 256)
        route_2 = net
        net = self.conv2d(net, 1024, 3, 2)
        for _ in range(4):
            net = self.res_block(net, 512)
        return route_1, route_2, net

    def yolo_block(self, x, filters):  # utils/layer_utils.py:71-79
        net = self.conv2d(x, filters, 1)
        net = self.conv2d(net, filters * 2, 3)
        net = self.conv2d(net, filters, 1)
        net = self.conv2d(net, filters * 2, 3)
        net = self.conv2d(net, filters, 1)
        route = net
        net = self.conv2d(net, filters * 2, 3)
        return route, net

    @staticmethod
    def upsample(x, out_hw):  # utils/layer_utils.py:82-87, [TF] align_corners=False
        h, w = x.shape[2], x.shape[3]
        assert out_hw[0] == 2 * h and out_hw[1] == 2 * w
        return x.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)


def forward(x_nhwc, params, class_num=80, is_training=False, emulate=None, bn_decay=0.999,
            dtype=torch.float32, as_torch=False, record=None):
    """model.py:30-80.  x_nhwc float32 [N,H,W,3] -> (fm1, fm2, fm3) NHWC.

    emulate in {None,'fp16','bf16'}: round the network input, every conv weight and
    every BN-conv output to that storage type (fp32 accumulate) — the storage model
    of the GPU engine; detection-head outputs stay fp32.
    Returns numpy arrays (or torch tensors, keeping the autograd graph, if as_torch).
    If is_training, also returns the list of updated (moving_mean, moving_var).
    """
    net = _Net(params, is_training, emulate, bn_decay, dtype, record)
    x = net._t(x_nhwc)
    x = _round_store(x, emulate)
    x = x.permute(0, 3, 1, 2)
    D = 3 * (5 + class_num)
    route_1, route_2, route_3 = net.darknet53_body(x)
    inter1, n1 = net.yolo_block(route_3, 512)                 # model.py:54
    fm1 = net.conv2d(n1, D, 1, bn=False)                      # model.py:55-58
    inter1 = net.conv2d(inter1, 256, 1)                       # model.py:60
    inter1 = net.upsample(inter1, route_2.shape[2:])          # model.py:61
    concat1 = torch.cat([inter1, route_2], dim=1)             # model.py:62
    inter2, n2 = net.yolo_block(concat1, 256)                 # model.py:64
    fm2 = net.conv2d(n2, D, 1, bn=False)                      # model.py:65-68
    inter2 = net.conv2d(inter2, 128, 1)                       # model.py:70
    inter2 = net.upsample(inter2, route_1.shape[2:])          # model.py:71
    concat2 = torch.cat([inter2, route_1], dim=1)             # model.py:72
    _, n3 = net.yolo_block(concat2, 128)                      # model.py:74
    fm3 = net.conv2d(n3, D, 1, bn=False)                      # model.py:75-78
    assert net.i == len(params) == 75
    fms = [t.permute(0, 2, 3, 1).contiguous() for t in (fm1, fm2, fm3)]
    if not as_torch:
        fms = [t.detach().numpy() for t in fms]
    if is_training:
        return tuple(fms), net.new_stats
    return tuple(fms)


# --------------------------------------------------------------------------------------
# Decode (model.py:82-190) — numpy float32, same op order as the TF graph
# --------------------------------------------------------------------------------------
def _sigmoid(x):
    x = np.asarray(x, dtype=F32)
    return (F32(1) / (F32(1) + np.exp(-x, dtype=F32))).astype(F32)


def reorg_layer(feature_map, anchors, img_size, class_num=80):
    """model.py:82-137.  feature_map [N,gh,gw,3*(5+C)], anchors [3,2] (w,h) px,
    img_size (H,W).  Returns x_y_offset[gh,gw,1,2], boxes[N,gh,gw,3,4] (cx,cy,w,h px),
    conf_logits[N,gh,gw,3,1], prob_logits[N,gh,gw,3,C]."""
    fm = np.asarray(feature_map, dtype=F32)
    gh, gw = fm.shape[1:3]
    ratio = (np.asarray(img_size, np.float64) / np.asarray([gh, gw], np.float64)).astype(F32)  # [h,w] :91
    anchors = np.asarray(anchors, F32)
    rescaled = np.stack([anchors[:, 0] / ratio[1], anchors[:, 1] / ratio[0]], axis=-1).astype(F32)  # :94
    fm = fm.reshape(-1, gh, gw, 3, 5 + class_num)                                   # :96
    centers, sizes, conf, prob = fm[..., 0:2], fm[..., 2:4], fm[..., 4:5], fm[..., 5:]  # :104
    centers = _sigmoid(centers)                                                     # :105
    gx, gy = np.meshgrid(np.arange(gw, dtype=np.int32), np.arange(gh, dtype=np.int32))  # :108-110
    xy_off = np.concatenate([gx.reshape(-1, 1), gy.reshape(-1, 1)], axis=-1)
    xy_off = xy_off.reshape(gh, gw, 1, 2).astype(F32)                               # :115
    centers = (centers + xy_off) * ratio[::-1]                                      # :118-120
    sizes = np.exp(sizes, dtype=F32) * rescaled                                     # :123
    sizes = sizes * ratio[::-1]                                                     # :126
    boxes = np.concatenate([centers, sizes], axis=-1).astype(F32)                   # :130
    return xy_off, boxes, conf, prob


def predict(feature_maps, anchors, img_size, class_num=80):
    """model.py:140-190 -> boxes[N,B,4] xyxy, confs[N,B,1], probs[N,B,C] float32."""
    anchors = np.asarray(anchors, F32)
    groups = [anchors[6:9], anchors[3:6], anchors[0:3]]                             # :147-149
    bl, cl, pl = [], [], []
    for fm, a in zip(feature_maps, groups):
        _, boxes, conf, prob = reorg_layer(fm, a, img_size, class_num)
        n = boxes.shape[0]
        bl.append(boxes.reshape(n, -1, 4))                                          # :155
        cl.append(_sigmoid(conf.reshape(n, -1, 1)))                                 # :156,167
        pl.append(_sigmoid(prob.reshape(n, -1, class_num)))                         # :157,168
    boxes = np.concatenate(bl, axis=1)                                              # :176-180
    confs = np.concatenate(cl, axis=1)
    probs = np.concatenate(pl, axis=1)
    cx, cy, w, h = boxes[..., 0:1], boxes[..., 1:2], boxes[..., 2:3], boxes[..., 3:4]
    half = F32(2)
    boxes = np.concatenate([cx - w / half, cy - h / half, cx + w / half, cy + h / half], axis=-1)  # :182-188
    return boxes.astype(F32), confs, probs


# --------------------------------------------------------------------------------------
# NMS (utils/nms_utils.py:8-48 + [TF] NonMaxSuppression CPU kernel)
# --------------------------------------------------------------------------------------
def tf_nms_cpu(boxes, scores, max_output_size, iou_threshold):
    """[TF] tf.image.non_max_suppression CPU kernel semantics (SURVEY.md B.4):
    descending score, ties -> lower index; select iff IoU with every already
    selected box is <= thr (strict > suppresses); float32 IoU with a true divide;
    corners normalised with min/max; area<=0 -> IoU 0.  Returns int32 indices."""
    boxes = np.asarray(boxes, F32).reshape(-1, 4)
    scores = np.asarray(scores, F32).reshape(-1)
    n = boxes.shape[0]
    if n == 0 or max_output_size <= 0:
        return np.zeros(0, np.int32)
    order = np.lexsort((np.arange(n), -scores.astype(np.float64)))  # stable: score desc, idx asc
    a0 = np.minimum(boxes[:, 0], boxes[:, 2]); a2 = np.maximum(boxes[:, 0], boxes[:, 2])
    a1 = np.minimum(boxes[:, 1], boxes[:, 3]); a3 = np.maximum(boxes[:, 1], boxes[:, 3])
    area = ((a2 - a0) * (a3 - a1)).astype(F32)
    thr = F32(iou_threshold)
    sel = []
    sx0 = np.empty(max_output_size, F32); sy0 = np.empty_like(sx0)
    sx1 = np.empty_like(sx0); sy1 = np.empty_like(sx0); sar = np.empty_like(sx0)
    for i in order:
        k = len(sel)
        if k >= max_output_size:
            break
        keep = True
        if k:
            ix0 = np.maximum(sx0[:k], a0[i]); iy0 = np.maximum(sy0[:k], a1[i])
            ix1 = np.minimum(sx1[:k], a2[i]); iy1 = np.minimum(sy1[:k], a3[i])
            inter = (np.maximum(ix1 - ix0, F32(0)) * np.maximum(iy1 - iy0, F32(0))).astype(F32)
            den = (sar[:k] + area[i] - inter).astype(F32)
            with np.errstate(divide="ignore", invalid="ignore"):
                iou = (inter / den).astype(F32)
            iou = np.where((sar[:k] <= 0) | (area[i] <= 0), F32(0), iou)
            keep = not bool(np.any(iou > thr))
        if keep:
            sx0[k], sy0[k], sx1[k], sy1[k], sar[k] = a0[i], a1[i], a2[i], a3[i], area[i]
            sel.append(i)
    return np.asarray(sel, np.int32)


def gpu_nms(boxes, scores, num_classes, max_boxes=50, score_thresh=0.5, nms_thresh=0.5, nms_fn=None):
    """utils/nms_utils.py:8-48 (single image).  Returns (boxes[K,4], score[K],
    label[K] int32, orig_index[K] int32) — the 4th output is the original box index
    (SURVEY.md F5), which the reference does not expose."""
    nms_fn = nms_fn or tf_nms_cpu
    boxes = np.asarray(boxes, F32).reshape(-1, 4)                 # :26
    score = np.asarray(scores, F32).reshape(-1, num_classes)     # :27
    mask = score >= F32(score_thresh)                            # :30
    bl, sl, ll, il = [], [], [], []
    for c in range(num_classes):                                 # :32
        pos = np.nonzero(mask[:, c])[0]
        fb = boxes[pos]                                          # :34
        fs = score[pos, c]                                       # :35
        idx = nms_fn(fb, fs, max_boxes, nms_thresh)              # :36-39
        bl.append(fb[idx]); sl.append(fs[idx])                   # :41-42
        ll.append(np.full(len(idx), c, np.int32))                # :40
        il.append(pos[idx].astype(np.int32))
    return (np.concatenate(bl, 0).reshape(-1, 4), np.concatenate(sl, 0),
            np.concatenate(ll, 0), np.concatenate(il, 0))


# ---- C restatement of the same NMS (oracle/nms_tf_cpu.c; built by `make -C oracle`) ----
_NMS_C = None


def _nms_c():
    global _NMS_C
    if _NMS_C is None:
        import ctypes, os
        path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libnms_oracle.so")
        if not os.path.exists(path):
            import subprocess
            subprocess.run(["make", "-C", os.path.dirname(path)], check=True, capture_output=True)
        lib = ctypes.CDLL(path)
        lib.yo_gpu_nms.restype = ctypes.c_int
        lib.yo_tf_nms.restype = ctypes.c_int
        _NMS_C = lib
    return _NMS_C


def gpu_nms_c(boxes, scores, num_classes, max_boxes=50, score_thresh=0.5, nms_thresh=0.5):
    """gpu_nms() through the C restatement (single thread).  Same outputs as gpu_nms()."""
    import ctypes
    lib = _nms_c()
    boxes = np.ascontiguousarray(boxes, F32).reshape(-1, 4)
    score = np.ascontiguousarray(scores, F32).reshape(-1, num_classes)
    B = boxes.shape[0]
    cap = max(num_classes * max_boxes, 1)
    ob = np.empty((cap, 4), F32); os_ = np.empty(cap, F32); ol = np.empty(cap, np.int32); oi = np.empty(cap, np.int32)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    k = lib.yo_gpu_nms(P(boxes), P(score), B, num_classes, int(max_boxes), ctypes.c_float(score_thresh),
                       ctypes.c_float(nms_thresh), P(ob), P(os_), P(ol), P(oi))
    return ob[:k].copy(), os_[:k].copy(), ol[:k].copy(), oi[:k].copy()


# --------------------------------------------------------------------------------------
# Loss (model.py:192-365) — torch (any float dtype) so autograd restates TF autodiff
# --------------------------------------------------------------------------------------
def _bce_logits(z, y):
    # [TF] sigmoid_cross_entropy_with_logits: max(z,0) - z*y + log(1+exp(-|z|))
    return torch.clamp(z, min=0) - z * y + torch.log1p(torch.exp(-torch.abs(z)))


def loss_layer(feature_map_i, y_true, anchors, img_size, class_num=80,
               use_label_smooth=False, use_focal_loss=False):
    """model.py:192-304.  torch tensors in, 4 scalar torch tensors out (xy, wh, conf, class)."""
    fm = feature_map_i
    dt = fm.dtype
    y_true = torch.as_tensor(y_true, dtype=dt)
    Nb, gh, gw = fm.shape[0], fm.shape[1], fm.shape[2]
    ratio = torch.tensor([img_size[0] / gh, img_size[1] / gw], dtype=dt)     # [h,w] :204
    N = float(Nb)                                                            # :206
    anchors_t = torch.as_tensor(np.asarray(anchors, F32), dtype=dt)
    # ---- reorg_layer (model.py:82-137) ----
    rescaled = torch.stack([anchors_t[:, 0] / ratio[1], anchors_t[:, 1] / ratio[0]], dim=-1)
    f = fm.reshape(Nb, gh, gw, 3, 5 + class_num)
    centers = torch.sigmoid(f[..., 0:2])
    gy, gx = torch.meshgrid(torch.arange(gh), torch.arange(gw), indexing="ij")
    xy_off = torch.stack([gx, gy], dim=-1).reshape(gh, gw, 1, 2).to(dt)
    rr = torch.stack([ratio[1], ratio[0]])                                   # ratio[::-1]
    pred_xy_px = (centers + xy_off) * rr
    pred_wh_px = torch.exp(f[..., 2:4]) * rescaled * rr
    pred_boxes = torch.cat([pred_xy_px, pred_wh_px], dim=-1)
    conf_logits = f[..., 4:5]
    prob_logits = f[..., 5:]

    object_mask = y_true[..., 4:5]                                           # :216
    # ignore mask, per image (:220-239); comparisons carry no gradient [TF]
    ign = []
    with torch.no_grad():
        for n in range(Nb):
            valid = y_true[n, ..., 0:4][object_mask[n, ..., 0] > 0]          # :224 boolean_mask
            if valid.shape[0] == 0:
                ign.append(torch.ones(gh, gw, 3, dtype=dt))                  # empty max -> -inf < 0.5 [TF]
                continue
            iou = box_iou(pred_boxes[n].detach(), valid)                     # :226
            best = iou.max(dim=-1).values                                    # :228
            ign.append((best < 0.5).to(dt))                                  # :230
    ignore_mask = torch.stack(ign, 0).unsqueeze(-1)                          # :237-239

    true_xy = y_true[..., 0:2] / rr - xy_off                                 # :248
    pred_xy = pred_xy_px / rr - xy_off                                       # :249
    true_twth = y_true[..., 2:4] / anchors_t                                 # :254
    pred_twth = pred_wh_px / anchors_t                                       # :255
    true_twth = torch.where(true_twth == 0, torch.ones_like(true_twth), true_twth)   # :257
    pred_twth = torch.where(pred_twth == 0, torch.ones_like(pred_twth), pred_twth)   # :259
    true_twth = torch.log(torch.clamp(true_twth, 1e-9, 1e9))                 # :261
    pred_twth = torch.log(torch.clamp(pred_twth, 1e-9, 1e9))                 # :262
    box_loss_scale = 2.0 - (y_true[..., 2:3] / float(img_size[1])) * (y_true[..., 3:4] / float(img_size[0]))  # :267
    mix_w = y_true[..., -1:]                                                 # :274
    xy_loss = torch.sum((true_xy - pred_xy) ** 2 * object_mask * box_loss_scale * mix_w) / N   # :276
    wh_loss = torch.sum((true_twth - pred_twth) ** 2 * object_mask * box_loss_scale * mix_w) / N  # :277
    conf_pos = object_mask                                                   # :280
    conf_neg = (1 - object_mask) * ignore_mask                               # :281
    bce = _bce_logits(conf_logits, object_mask)
    conf_loss = conf_pos * bce + conf_neg * bce                              # :282-285
    if use_focal_loss:                                                       # :286-291
        focal = torch.abs(object_mask - torch.sigmoid(conf_logits)) ** 2.0
        conf_loss = conf_loss * focal
    conf_loss = torch.sum(conf_loss * mix_w) / N                             # :292
    if use_label_smooth:                                                     # :296-300
        label_target = (1 - 0.01) * y_true[..., 5:-1] + 0.01 * 1.0 / class_num
    else:
        label_target = y_true[..., 5:-1]
    class_loss = object_mask * _bce_logits(prob_logits, label_target) * mix_w  # :301
    class_loss = torch.sum(class_loss) / N                                   # :302
    return xy_loss, wh_loss, conf_loss, class_loss


def box_iou(pred_boxes, valid_true_boxes):
    """model.py:307-345: centre-format IoU [gh,gw,3,4] x [V,4] -> [gh,gw,3,V]."""
    pxy = pred_boxes[..., 0:2].unsqueeze(-2)
    pwh = pred_boxes[..., 2:4].unsqueeze(-2)
    txy = valid_true_boxes[:, 0:2]
    twh = valid_true_boxes[:, 2:4]
    mins = torch.maximum(pxy - pwh / 2.0, txy - twh / 2.0)
    maxs = torch.minimum(pxy + pwh / 2.0, txy + twh / 2.0)
    wh = torch.clamp(maxs - mins, min=0.0)
    inter = wh[..., 0] * wh[..., 1]
    parea = pwh[..., 0] * pwh[..., 1]
    tarea = (twh[..., 0] * twh[..., 1]).unsqueeze(0)
    return inter / (parea + tarea - inter + 1e-10)


def compute_loss(y_pred, y_true, anchors, img_size, class_num=80,
                 use_label_smooth=False, use_focal_loss=False):
    """model.py:348-365 -> [total, xy, wh, conf, class] (torch scalars)."""
    anchors = np.asarray(anchors, F32)
    groups = [anchors[6:9], anchors[3:6], anchors[0:3]]
    acc = [0.0, 0.0, 0.0, 0.0]
    for i in range(3):
        fm = y_pred[i] if isinstance(y_pred[i], torch.Tensor) else torch.from_numpy(np.asarray(y_pred[i]))
        r = loss_layer(fm, y_true[i], groups[i], img_size, class_num, use_label_smooth, use_focal_loss)
        for j in range(4):
            acc[j] = acc[j] + r[j]
    total = acc[0] + acc[1] + acc[2] + acc[3]
    return [total] + acc


def loss_and_grad(y_pred, y_true, anchors, img_size, class_num=80, use_label_smooth=False,
                  use_focal_loss=False, dtype=torch.float32):
    """Loss values and d(total)/d(feature_map_i) as TF autodiff would produce them."""
    fms = [torch.tensor(np.asarray(f), dtype=dtype, requires_grad=True) for f in y_pred]
    losses = compute_loss(fms, y_true, anchors, img_size, class_num, use_label_smooth, use_focal_loss)
    losses[0].backward()
    return [float(l.detach()) for l in losses], [f.grad.numpy() for f in fms]


# --------------------------------------------------------------------------------------
# y_true builder (utils/data_utils.py:51-115) — restated; pinned by golden vectors
# --------------------------------------------------------------------------------------
def process_box(boxes, labels, img_size, class_num, anchors):
    """boxes [V,5] (x0,y0,x1,y1,mix_w) f32, labels [V] int; img_size (W,H) like the
    reference (utils/data_utils.py:72-74 index [1] for rows).  Returns 3 arrays."""
    boxes = np.asarray(boxes, F32)
    anchors = np.asarray(anchors, F32)
    anchors_mask = [[6, 7, 8], [3, 4, 5], [0, 1, 2]]
    centers = (boxes[:, 0:2] + boxes[:, 2:4]) / 2
    sizes = boxes[:, 2:4] - boxes[:, 0:2]
    ys = []
    for s in (32, 16, 8):
        y = np.zeros((img_size[1] // s, img_size[0] // s, 3, 6 + class_num), F32)
        y[..., -1] = 1.0
        ys.append(y)
    bs = np.expand_dims(sizes, 1)
    mins = np.maximum(-bs / 2, -anchors / 2)
    maxs = np.minimum(bs / 2, anchors / 2)
    whs = maxs - mins
    iou = (whs[:, :, 0] * whs[:, :, 1]) / (
        bs[:, :, 0] * bs[:, :, 1] + anchors[:, 0] * anchors[:, 1] - whs[:, :, 0] * whs[:, :, 1] + 1e-10)
    best = np.argmax(iou, axis=1)
    for i, idx in enumerate(best):
        g = 2 - idx // 3
        ratio = {0: 32.0, 1: 16.0, 2: 8.0}[g]
        x = int(np.floor(centers[i, 0] / ratio))
        y = int(np.floor(centers[i, 1] / ratio))
        k = anchors_mask[g].index(idx)
        c = int(labels[i])
        ys[g][y, x, k, :2] = centers[i]
        ys[g][y, x, k, 2:4] = sizes[i]
        ys[g][y, x, k, 4] = 1.0
        ys[g][y, x, k, 5 + c] = 1.0
        ys[g][y, x, k, -1] = boxes[i, -1]
    return ys[0], ys[1], ys[2]


def synth_gt(rng, img_w, img_h, class_num=80, max_boxes=50):
    """SURVEY.md §8d cfg 3 ground truth for one image: boxes [V,5], labels [V]."""
    v = int(rng.integers(1, max_boxes + 1))
    w = np.exp(rng.uniform(np.log(8), np.log(400), v))
    h = np.exp(rng.uniform(np.log(8), np.log(400), v))
    cx = rng.uniform(0, img_w, v); cy = rng.uniform(0, img_h, v)
    x0 = np.clip(cx - w / 2, 0, img_w - 1); x1 = np.clip(cx + w / 2, 1, img_w)
    y0 = np.clip(cy - h / 2, 0, img_h - 1); y1 = np.clip(cy + h / 2, 1, img_h)
    x1 = np.maximum(x1, x0 + 1); y1 = np.maximum(y1, y0 + 1)
    boxes = np.stack([x0, y0, x1, y1, np.ones(v)], axis=1).astype(F32)
    labels = rng.integers(0, class_num, v).astype(np.int64)
    return boxes, labels


# --------------------------------------------------------------------------------------
# Training step (train.py:105-115, utils/misc_utils.py:151-153)
# --------------------------------------------------------------------------------------
def train_step(x_nhwc, y_true, params, velocity, lr, anchors, class_num=80, use_label_smooth=False,
               use_focal_loss=False, bn_decay=0.99, weight_decay=5e-4, momentum=0.9, clip=100.0,
               emulate=None, dtype=torch.float32, optimizer="momentum", decay=0.9, beta1=0.9, beta2=0.999,
               epsilon=None, slot2=None, step=0, freeze_bn=False, trainable=None):
    """One reference training step on CPU.  Returns (losses, grads, new_params, new_velocity) — for rmsprop / adam
    new_velocity is a pair (slot1, slot2) of per-layer dicts.

    grads are d(total + l2)/d(param) *before* clipping, keyed like params
    ('w','gamma','beta','b'); L2 = wd * sum(w^2)/2 on conv weights only (model.py:49).
    optimizer (utils/misc_utils.py:151-161, [TF] TensorFlow 1.x update rules):
      momentum  v = m*v + g; w -= lr*v                                  (MomentumOptimizer, no Nesterov)
      sgd       w -= lr*g                                               (GradientDescentOptimizer)
      rmsprop   ms = d*ms + (1-d)g^2 (ms starts at 1); mom = m*mom + lr*g/sqrt(ms+1e-10); w -= mom
      adam      t = step+1; lr_t = lr*sqrt(1-b2^t)/(1-b1^t); m = b1*m+(1-b1)g; v = b2*v+(1-b2)g^2; w -= lr_t*m/(sqrt(v)+1e-8)
    `velocity` is slot 1 (momentum / rmsprop mom / adam m), `slot2` the rmsprop ms / adam v (None: TF's initial value).
    freeze_bn: the graph built with is_training=False (train.py:72): BN uses and keeps its moving statistics.
    trainable: optional set of conv indices in update_vars (train.py:81); others are left untouched.
    """
    if epsilon is None:
        epsilon = 1e-10 if optimizer == "rmsprop" else 1e-8
    tp = []
    for p in params:
        q = {}
        for k, v in p.items():
            t = torch.tensor(np.asarray(v), dtype=dtype)
            if k in ("w", "gamma", "beta", "b"):
                t.requires_grad_(True)
            q[k] = t
        tp.append(q)
    H, W = x_nhwc.shape[1:3]
    out = forward(torch.tensor(x_nhwc, dtype=dtype), tp, class_num, not freeze_bn, emulate, bn_decay, dtype, as_torch=True)
    fms, new_stats = (out, None) if freeze_bn else out       # forward() returns the moving statistics only when training
    losses = compute_loss(list(fms), y_true, anchors, (H, W), class_num, use_label_smooth, use_focal_loss)
    l2 = sum((q["w"] ** 2).sum() for q in tp) * (weight_decay / 2.0)        # train.py:78
    (losses[0] + l2).backward()                                              # train.py:112
    grads, new_params, new_vel, new_s2 = [], [], [], []
    si = 0
    for li, (q, p, v) in enumerate(zip(tp, params, velocity)):
        g, npar, nv, n2 = {}, {}, {}, {}
        for k in q:
            if q[k].requires_grad:
                gk = q[k].grad
                g[k] = gk.numpy().copy()
                if trainable is not None and li not in trainable:
                    continue
                nrm = torch.sqrt((gk * gk).sum())
                gc = gk * clip / torch.clamp(nrm, min=clip)                  # train.py:113-114 clip_by_norm
                s1 = torch.as_tensor(v[k], dtype=dtype)
                if optimizer == "momentum":                                  # utils/misc_utils.py:153
                    vk = momentum * s1 + gc
                    nv[k] = vk.numpy()
                    npar[k] = (q[k].detach() - lr * vk).numpy()
                elif optimizer == "sgd":                                     # :159
                    nv[k] = s1.numpy()
                    npar[k] = (q[k].detach() - lr * gc).numpy()
                elif optimizer == "rmsprop":                                 # :155
                    ms0 = torch.ones_like(gc) if slot2 is None else torch.as_tensor(slot2[li][k], dtype=dtype)
                    ms = decay * ms0 + (1 - decay) * gc * gc
                    mom = momentum * s1 + lr * gc / torch.sqrt(ms + epsilon)
                    nv[k], n2[k] = mom.numpy(), ms.numpy()
                    npar[k] = (q[k].detach() - mom).numpy()
                elif optimizer == "adam":                                    # :157
                    v0 = torch.zeros_like(gc) if slot2 is None else torch.as_tensor(slot2[li][k], dtype=dtype)
                    t = step + 1
                    lr_t = lr * math.sqrt(1 - beta2 ** t) / (1 - beta1 ** t)
                    m1 = beta1 * s1 + (1 - beta1) * gc
                    v1 = beta2 * v0 + (1 - beta2) * gc * gc
                    nv[k], n2[k] = m1.numpy(), v1.numpy()
                    npar[k] = (q[k].detach() - lr_t * m1 / (torch.sqrt(v1) + epsilon)).numpy()
                else:
                    raise ValueError("Unsupported optimizer type!")          # :161
        if "gamma" in q and not freeze_bn:
            mm, mv = new_stats[si]; si += 1
            npar["mean"], npar["var"] = mm.numpy(), mv.numpy()
        grads.append(g); new_params.append(npar); new_vel.append(nv); new_s2.append(n2)
    out_vel = new_vel if optimizer in ("momentum", "sgd") else (new_vel, new_s2)
    return [float(l.detach()) for l in losses] + [float(l2.detach())], grads, new_params, out_vel


# --------------------------------------------------------------------------------------
# Learning-rate schedules (utils/misc_utils.py:129-148, warm-up train.py:93-99)
# --------------------------------------------------------------------------------------
def learning_rate(args, global_step):
    """The value of train.py:93-99's `learning_rate` tensor at float `global_step`.  `args` carries the fields of
    args.py (lr_type, learning_rate_init, lr_decay_freq, lr_decay_factor, lr_lower_bound, total_epoches,
    use_warm_up, warm_up_epoch, train_batch_num, pw_boundaries, pw_values).  [TF] semantics restated:
      exponential_decay(staircase): lr0 * factor ** floor(step / freq), then max(., lower bound)
      cosine_decay_restarts(t_mul=2, m_mul=1, alpha=0): first period = freq, each next one twice as long
      piecewise_constant: values[i] for boundaries[i-1] < step <= boundaries[i]  (x <= b[0] -> v[0])"""
    gs = float(global_step)
    if args.use_warm_up:
        wu = args.train_batch_num * args.warm_up_epoch
        if gs < wu:
            return args.learning_rate_init * gs / wu                         # train.py:95
        gs = gs - wu                                                         # train.py:96
    t = args.lr_type
    if t == "exponential":
        return max(args.learning_rate_init * args.lr_decay_factor ** math.floor(gs / args.lr_decay_freq), args.lr_lower_bound)
    if t == "cosine_decay":
        train_steps = (args.total_epoches - float(args.use_warm_up) * args.warm_up_epoch) * args.train_batch_num
        return args.lr_lower_bound + 0.5 * (args.learning_rate_init - args.lr_lower_bound) * (1 + math.cos(gs / train_steps * math.pi))
    if t == "cosine_decay_restart":
        frac = gs / args.lr_decay_freq
        i = math.floor(math.log(1.0 - frac * (1.0 - 2.0)) / math.log(2.0))  # [TF] compute_step, t_mul = 2
        frac = (frac - (1.0 - 2.0 ** i) / (1.0 - 2.0)) / 2.0 ** i
        return args.learning_rate_init * 0.5 * (1.0 + math.cos(math.pi * frac))
    if t == "fixed":
        return args.learning_rate_init
    if t == "piecewise":
        for b, v in zip(args.pw_boundaries, args.pw_values):
            if gs <= b:
                return v
        return args.pw_values[-1]
    raise ValueError("Unsupported learning rate type!")


# --------------------------------------------------------------------------------------
# Darknet .weights stream (utils/misc_utils.py:70-126)
# --------------------------------------------------------------------------------------
def write_darknet_weights(path, params):
    """Inverse of load_weights: 5 x int32 header, then per conv [beta,gamma,mean,var]
    or [bias], then weights as (Cout,Cin,kh,kw) float32."""
    with open(path, "wb") as f:
        np.array([0, 2, 0, 0, 0], np.int32).tofile(f)
        for p in params:
            if "gamma" in p:
                for k in ("beta", "gamma", "mean", "var"):                  # :93
                    np.asarray(p[k], F32).tofile(f)
            else:
                np.asarray(p["b"], F32).tofile(f)                           # :102-108
            np.ascontiguousarray(np.transpose(p["w"], (3, 2, 0, 1)), F32).tofile(f)  # inverse of :117-120


def load_darknet_weights(path, class_num=80):
    """utils/misc_utils.py:70-126 restated against conv_specs() creation order."""
    with open(path, "rb") as f:
        np.fromfile(f, dtype=np.int32, count=5)                             # :78
        ws = np.fromfile(f, dtype=np.float32)                               # :79
    ptr = 0
    params = []
    for _, cin, cout, k, s, bn in conv_specs(class_num):
        p = {}
        if bn:
            for name in ("beta", "gamma", "mean", "var"):                   # :92-99
                p[name] = ws[ptr:ptr + cout].copy(); ptr += cout
        else:
            p["b"] = ws[ptr:ptr + cout].copy(); ptr += cout                 # :102-110
        n = k * k * cin * cout
        w = ws[ptr:ptr + n].reshape(cout, cin, k, k); ptr += n              # :114-118
        p["w"] = np.ascontiguousarray(np.transpose(w, (2, 3, 1, 0)))        # :120
        params.append(p)
    assert ptr == ws.size, (ptr, ws.size)
    return params


# --------------------------------------------------------------------------------------
# Pre-processing (utils/data_aug.py:274-293 letterbox_resize with interp=0; test_single_image.py:44-46)
# --------------------------------------------------------------------------------------
def letterbox_preprocess(img_bgr_u8, new_width, new_height):
    """letterbox_resize(img, new_width, new_height, interp=0) -> cvtColor(BGR2RGB) -> float32 / 255, in numpy.
    [TF-free] OpenCV's nearest-neighbour resize restated: src index = min(floor(dst * (1 / (dst_size / src_size))),
    src_size - 1), computed in double (modules/imgproc/src/resize.cpp: resizeNN).
    Returns (x [1, new_height, new_width, 3] float32 RGB in [0, 1], resize_ratio, dw, dh)."""
    img = np.asarray(img_bgr_u8, np.uint8)
    ori_h, ori_w = img.shape[:2]
    ratio = min(new_width / ori_w, new_height / ori_h)                            # :280
    rw, rh = int(ratio * ori_w), int(ratio * ori_h)                               # :282-283
    ifx, ify = 1.0 / (rw / ori_w), 1.0 / (rh / ori_h)
    sx = np.minimum(np.floor(np.arange(rw) * ifx).astype(np.int64), ori_w - 1)
    sy = np.minimum(np.floor(np.arange(rh) * ify).astype(np.int64), ori_h - 1)
    resized = img[sy][:, sx]                                                      # cv2.resize(..., interpolation=0)
    padded = np.full((new_height, new_width, 3), 128, np.uint8)                   # :286
    dw, dh = int((new_width - rw) / 2), int((new_height - rh) / 2)                # :288-289
    padded[dh: rh + dh, dw: rw + dw, :] = resized                                 # :291
    x = padded[..., ::-1].astype(F32)                                             # BGR -> RGB, np.asarray(img, np.float32)
    return (x[np.newaxis] / F32(255.0)).astype(F32), ratio, dw, dh
