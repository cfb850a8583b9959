"""A numpy/torch-CPU backed stand-in for the handful of `tensorflow` 1.x symbols that
the reference's {model.py,utils/layer_utils.py,utils/nms_utils.py,utils/misc_utils.py,
utils/data_utils.py} touch, so that the reference's *own Python sources* can be
executed in this container (TensorFlow itself is not installable here).

TEST INFRASTRUCTURE ONLY (used by make_golden.py to generate tests/golden/*.npz).
It executes eagerly: every "tensor" is a float32/int32 numpy array.  The TF *kernel*
semantics it has to supply itself (conv2d, fused batch norm, non_max_suppression,
sigmoid_cross_entropy_with_logits, resize_nearest_neighbor) are restated from
SURVEY.md Appendix B and marked [TF] — those remain unpinned; what the golden
vectors pin is everything the reference wrote in Python on top of them.
"""
from __future__ import annotations

import contextlib
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

float32 = np.float32
int32 = np.int32


def _dt(d):
    if d in ("bool", bool):
        return np.bool_
    if d in ("int32", int32):
        return np.int32
    if d in ("float32", float32):
        return np.float32
    return d


# ---- basic ops -----------------------------------------------------------------------
def shape(x):
    return np.array(np.shape(x), dtype=np.int32)


def cast(x, dtype):
    return np.asarray(x).astype(_dt(dtype))


def reshape(x, s):
    return np.reshape(x, [int(v) for v in s])


def split(x, sizes, axis=-1):
    idx = np.cumsum(sizes)[:-1]
    return np.split(x, idx, axis=axis)


def concat(xs, axis):
    return np.concatenate(xs, axis=axis)


def sigmoid(x):
    x = np.asarray(x, np.float32)
    return (np.float32(1) / (np.float32(1) + np.exp(-x, dtype=np.float32))).astype(np.float32)


def exp(x):
    return np.exp(np.asarray(x, np.float32), dtype=np.float32)


def log(x):
    return np.log(np.asarray(x, np.float32), dtype=np.float32)


def range_(n, dtype=np.int32):
    return np.arange(int(n), dtype=_dt(dtype))


def meshgrid(a, b):
    return np.meshgrid(a, b)


def expand_dims(x, axis):
    return np.expand_dims(x, axis)


def maximum(a, b):
    return np.maximum(a, b)


def minimum(a, b):
    return np.minimum(a, b)


def reduce_max(x, axis=None):
    x = np.asarray(x)
    if axis is not None and x.shape[axis] == 0:   # [TF] empty max -> lowest float
        out = list(x.shape); del out[axis]
        return np.full(out, np.finfo(np.float32).min, np.float32)
    return np.max(x, axis=axis)


def reduce_sum(x, axis=None):
    return np.sum(np.asarray(x, np.float32), axis=axis, dtype=np.float32)


def square(x):
    return np.square(x)


def where(condition, x, y):
    return np.where(condition, x, y)


def equal(a, b):
    return np.equal(a, b)


def less(a, b):
    return np.less(a, b)


def greater_equal(a, b):
    return np.greater_equal(a, b)


def ones_like(x, dtype=None):
    return np.ones_like(x, dtype=_dt(dtype) if dtype is not None else None)


def clip_by_value(x, lo, hi):
    return np.clip(x, np.float32(lo), np.float32(hi))


def pow_(x, y):
    return np.power(x, np.float32(y))


def abs_(x):
    return np.abs(x)


def boolean_mask(x, mask):
    return np.asarray(x)[np.asarray(mask, bool)]


def gather(x, idx):
    return np.asarray(x)[np.asarray(idx, np.int64)]


def constant(v, dtype=None):
    if dtype is None:
        return np.float32(v) if isinstance(v, float) else np.asarray(v)
    return np.asarray(v, dtype=_dt(dtype))


def identity(x, name=None):
    return x


def pad(x, paddings, mode="CONSTANT"):
    return np.pad(x, paddings, mode="constant")


class TensorArray:
    def __init__(self, dtype, size=0, dynamic_size=True):
        self.items = {}

    def write(self, idx, v):
        self.items[int(idx)] = v
        return self

    def stack(self):
        return np.stack([self.items[i] for i in sorted(self.items)], axis=0)


def while_loop(cond, body, loop_vars):
    v = list(loop_vars)
    while bool(cond(*v)):
        v = list(body(*v))
    return v


@contextlib.contextmanager
def variable_scope(name, *a, **k):
    yield


def zeros_initializer():
    return "zeros"


# ---- tf.nn ---------------------------------------------------------------------------
def leaky_relu(x, alpha=0.2):
    return np.maximum(x, np.float32(alpha) * x)  # [TF]


def sigmoid_cross_entropy_with_logits(labels=None, logits=None):
    z = np.asarray(logits, np.float32); y = np.asarray(labels, np.float32)
    # [TF] max(x,0) - x*z + log(1+exp(-|x|))
    return (np.maximum(z, 0) - z * y + np.log1p(np.exp(-np.abs(z)))).astype(np.float32)


# ---- tf.image ------------------------------------------------------------------------
def resize_nearest_neighbor(x, size, name=None):
    h, w = int(size[0]), int(size[1])
    ih, iw = x.shape[1], x.shape[2]
    yi = np.floor(np.arange(h) * (ih / h)).astype(np.int64)  # [TF] align_corners=False
    xi = np.floor(np.arange(w) * (iw / w)).astype(np.int64)
    return x[:, yi][:, :, xi]


_NMS_IMPL = {"fn": None}


def non_max_suppression(boxes=None, scores=None, max_output_size=None, iou_threshold=0.5, name=None):
    return _NMS_IMPL["fn"](boxes, scores, int(max_output_size), float(iou_threshold))


# ---- tf.contrib.slim -----------------------------------------------------------------
class _Slim:
    def __init__(self):
        self.scopes = []        # stack of (set(func names), kwargs)
        self.weights = None     # iterator over per-conv param dicts (creation order)
        self.updated_stats = []

    @contextlib.contextmanager
    def arg_scope(self, funcs, **kwargs):
        self.scopes.append(({f.__name__ for f in funcs}, kwargs))
        try:
            yield
        finally:
            self.scopes.pop()

    def _defaults(self, name):
        d = {}
        for names, kw in self.scopes:
            if name in names:
                d.update(kw)
        return d

    def l2_regularizer(self, scale):
        return lambda w: np.float32(scale) * np.sum(np.square(w)) / np.float32(2)

    def batch_norm(self, x, p, decay=0.999, epsilon=0.001, scale=False, center=True,
                   is_training=True, fused=None, reuse=None):
        # [TF] fused batch norm (SURVEY.md B.1)
        if is_training:
            mean = x.mean(axis=(0, 1, 2), dtype=np.float64)
            var = x.var(axis=(0, 1, 2), dtype=np.float64)
            n = x.size // x.shape[-1]
            self.updated_stats.append((
                (p["mean"] * decay + (1 - decay) * mean).astype(np.float32),
                (p["var"] * decay + (1 - decay) * var * n / max(n - 1, 1)).astype(np.float32)))
            mean = mean.astype(np.float32); var = var.astype(np.float32)
        else:
            mean, var = p["mean"], p["var"]
        g = p["gamma"] if scale else np.float32(1)
        inv = (g / np.sqrt(var + np.float32(epsilon))).astype(np.float32)
        return (x * inv + (p["beta"] - mean * inv)).astype(np.float32)

    def conv2d(self, inputs, num_outputs, kernel_size, stride=1, padding="SAME", **kw):
        d = dict(normalizer_fn=None, normalizer_params=None, activation_fn=lambda t: np.maximum(t, 0),
                 biases_initializer="zeros", weights_regularizer=None, reuse=None)
        d.update(self._defaults("conv2d")); d.update(kw)
        p = next(self.weights)
        w = p["w"]
        k = int(kernel_size)
        assert w.shape == (k, k, inputs.shape[-1], num_outputs), (w.shape, inputs.shape, num_outputs)
        x = torch.from_numpy(np.ascontiguousarray(inputs, dtype=np.float32)).permute(0, 3, 1, 2)
        wt = torch.from_numpy(np.ascontiguousarray(w)).permute(3, 2, 0, 1)
        if padding == "SAME":   # [TF] stride-1 SAME for odd k == symmetric k//2
            assert stride == 1
            pd = k // 2
        else:
            pd = 0
        y = F.conv2d(x, wt, None, stride=stride, padding=pd).permute(0, 2, 3, 1).contiguous().numpy()
        if d["normalizer_fn"] is not None:
            bn_kw = dict(self._defaults("batch_norm")); bn_kw.update(d["normalizer_params"] or {})
            bn_kw.pop("reuse", None)
            y = self.batch_norm(y, p, **bn_kw)
        elif d["biases_initializer"] is not None:
            y = y + p["b"]
        if d["activation_fn"] is not None:
            y = d["activation_fn"](y)
        return y.astype(np.float32)


def install(nms_fn):
    """Put the shim into sys.modules as `tensorflow`; returns (tf_module, slim)."""
    _NMS_IMPL["fn"] = nms_fn
    tf = types.ModuleType("tensorflow")
    for name, fn in dict(
        shape=shape, cast=cast, reshape=reshape, split=split, concat=concat, sigmoid=sigmoid, exp=exp, log=log,
        meshgrid=meshgrid, expand_dims=expand_dims, maximum=maximum, minimum=minimum, reduce_max=reduce_max,
        reduce_sum=reduce_sum, square=square, where=where, equal=equal, less=less, greater_equal=greater_equal,
        ones_like=ones_like, clip_by_value=clip_by_value, boolean_mask=boolean_mask, gather=gather,
        constant=constant, identity=identity, pad=pad, TensorArray=TensorArray, while_loop=while_loop,
        variable_scope=variable_scope, zeros_initializer=zeros_initializer, float32=float32, int32=int32,
    ).items():
        setattr(tf, name, fn)
    setattr(tf, "range", range_)
    setattr(tf, "pow", pow_)
    setattr(tf, "abs", abs_)
    nn = types.ModuleType("tensorflow.nn")
    nn.sigmoid = sigmoid
    nn.leaky_relu = leaky_relu
    nn.sigmoid_cross_entropy_with_logits = sigmoid_cross_entropy_with_logits
    tf.nn = nn
    image = types.ModuleType("tensorflow.image")
    image.resize_nearest_neighbor = resize_nearest_neighbor
    image.non_max_suppression = non_max_suppression
    tf.image = image
    slim = _Slim()
    contrib = types.ModuleType("tensorflow.contrib")
    contrib.slim = slim
    tf.contrib = contrib
    core = types.ModuleType("tensorflow.core")
    fw = types.ModuleType("tensorflow.core.framework")
    spb = types.ModuleType("tensorflow.core.framework.summary_pb2")
    core.framework = fw
    fw.summary_pb2 = spb
    tf.core = core
    sys.modules.update({
        "tensorflow": tf, "tensorflow.nn": nn, "tensorflow.image": image, "tensorflow.contrib": contrib,
        "tensorflow.core": core, "tensorflow.core.framework": fw, "tensorflow.core.framework.summary_pb2": spb,
    })
    return tf, slim
