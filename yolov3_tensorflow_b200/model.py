"""`yolov3` — the reference's model class (model.py:12-365 of wizyoung/YOLOv3_TensorFlow)
re-hosted on the H100 engine.

Same constructor and method names/arguments as the reference.  The reference methods
build TF1 graph nodes; these run eagerly: they take/return CUDA `torch.Tensor`s (used
purely as device-buffer containers, NHWC, float32 at the API surface) and enqueue
hand-written sm_90a kernels from libyolob200.so on the current CUDA stream.
There is no torch op on the compute path and no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from ._lib import lib, check, ptr, stream_handle


def _dtype_code(dtype):
    if dtype in ("fp16", "float16", torch.float16, _lib.YB_F16):
        return _lib.YB_F16, torch.float16
    if dtype in ("bf16", "bfloat16", torch.bfloat16, _lib.YB_BF16):
        return _lib.YB_BF16, torch.bfloat16
    raise ValueError(f"unsupported compute dtype {dtype!r} (fp16 or bf16)")


def _as_cuda_f32(x, device):
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
    if not isinstance(x, torch.Tensor):
        raise TypeError(f"expected a torch.Tensor or numpy array, got {type(x)}")
    if x.dtype != torch.float32:
        raise TypeError(f"expected float32, got {x.dtype}")
    if not x.is_cuda:
        x = x.to(device, non_blocking=True)
    return x.contiguous()


class _Plan:
    """One yb_net (fixed batch/H/W): its own activation arena, bound to the MODEL's parameter arena.

    The parameter-arena layout depends only on (class_num, dtype, training) (include/yolob200.h: yb_net_bind), so all
    plans of a model share one arena: one set of master weights / 16-bit copies / folded BN and ONE optimizer state,
    whatever batch size or resolution a step runs at (the reference's single MomentumOptimizer under
    multi_scale_train, train.py:47-49)."""

    def __init__(self, model, n, h, w, training=False):
        self.n, self.h, self.w = n, h, w
        self.training = training
        self.act_dtype = model._torch_dtype
        self.handle = C.c_void_p()
        check(lib.yb_net_create(C.byref(self.handle), model.class_num, n, h, w, model._dtype_code, int(training)), "yb_net_create")
        a, p = C.c_size_t(), C.c_size_t()
        check(lib.yb_net_arena_bytes(self.handle, C.byref(a), C.byref(p)), "yb_net_arena_bytes")
        self.param_bytes = p.value
        dev = model.device
        self.act = torch.zeros(max(a.value, 256), dtype=torch.uint8, device=dev)
        self.par = None
        self.num_layers = lib.yb_net_num_layers(self.handle)
        self.loss4 = torch.zeros(4, dtype=torch.float64, device=dev) if training else None

    def bind(self, par):
        self.par = par
        check(lib.yb_net_bind(self.handle, ptr(self.act), self.act.numel(), ptr(par), par.numel(), stream_handle()), "yb_net_bind")

    def _view(self, p, shape, dtype=torch.float32):
        """torch view of `shape` floats at device pointer p inside the parameter arena."""
        off = p - self.par.data_ptr()
        n = int(np.prod(shape))
        return self.par[off: off + n * 4].view(dtype).view(*shape)

    def conv_params(self, i):
        """Views of layer i's float32 master parameters: dict(w [cout,k,k,cin] OHWI, gamma, beta, mean, var | b)."""
        ps = [C.c_void_p() for _ in range(6)]
        check(lib.yb_net_get_conv_params(self.handle, i, *[C.byref(q) for q in ps]), "yb_net_get_conv_params")
        info = self.layer_info(i)
        out = {"w": self._view(ps[0].value, (info.cout, info.ksize, info.ksize, info.cin))}
        for name, q in zip(("gamma", "beta", "mean", "var", "b"), ps[1:]):
            if q.value:
                out[name] = self._view(q.value, (info.cout,))
        return out

    def layer_grads(self, i):
        ps = [C.c_void_p() for _ in range(4)]
        check(lib.yb_net_layer_grad(self.handle, i, *[C.byref(q) for q in ps]), "yb_net_layer_grad")
        info = self.layer_info(i)
        out = {"w": self._view(ps[0].value, (info.cout, info.ksize, info.ksize, info.cin))}
        for name, q in zip(("gamma", "beta", "b"), ps[1:]):
            if q.value:
                out[name] = self._view(q.value, (info.cout,))
        return out

    def train_buffer(self, i, which):
        """Strided view [n,h,w,c] of layer i's training scratch: which = 'z' | 'dz' | 'dA' | 'in' | 'dX' (the gradient
        w.r.t. the layer input, which its dgrad writes), or the layer's 16-bit forward weights 'w16' as [cout_pad,
        k*k*cin] (parameter arena)."""
        code = {"z": 0, "dz": 1, "dA": 2, "in": 3, "dX": 5, "w16": 6}[which]
        p, ld, hh, ww = C.c_void_p(), C.c_int(), C.c_int(), C.c_int()
        check(lib.yb_net_train_buffer(self.handle, i, code, C.byref(p), C.byref(ld), C.byref(hh), C.byref(ww)), "yb_net_train_buffer")
        tdt = torch.float16 if self.act_dtype == torch.float16 else torch.bfloat16
        if which == "w16":
            off = p.value - self.par.data_ptr()
            return self.par[off: off + hh.value * ld.value * 2].view(tdt).view(hh.value, ld.value)
        info = self.layer_info(i)
        c = info.cin if which in ("in", "dX") else info.cout
        off = p.value - self.act.data_ptr()
        h, w = hh.value, ww.value
        nelem = (self.n * h * w - 1) * ld.value + c
        flat = self.act[off: off + nelem * 2].view(tdt)
        return flat.as_strided((self.n, h, w, c), (h * w * ld.value, w * ld.value, ld.value, 1))

    def dgrad_weights(self, i):
        """Layer i's 16-bit dgrad weights (flip + transpose of the masters, csrc/optim.cu), flat [cin_pad * k * k * k_cout]."""
        p, ld, hh, ww = C.c_void_p(), C.c_int(), C.c_int(), C.c_int()
        check(lib.yb_net_train_buffer(self.handle, i, 4, C.byref(p), C.byref(ld), C.byref(hh), C.byref(ww)), "yb_net_train_buffer")
        off = p.value - self.par.data_ptr()
        tdt = torch.float16 if self.act_dtype == torch.float16 else torch.bfloat16
        return self.par[off: off + hh.value * ww.value * ld.value * 2].view(tdt)

    def grad_range(self, first_layer, last_layer):
        """Flat-gradient slice owned by layers [first_layer, last_layer] (a data-parallel bucket)."""
        p, n = C.c_void_p(), C.c_size_t()
        check(lib.yb_net_grad_range(self.handle, int(first_layer), int(last_layer), C.byref(p), C.byref(n)), "yb_net_grad_range")
        return self._view(p.value, (n.value,))

    def bn_exchange_buffer(self, i, backward):
        """Layer i's sync-BN exchange slab (float32 [2 * cout_pad], activation arena): forward [Σz | Σz²], backward
        [Σdact·ẑ | Σdact]."""
        p, n = C.c_void_p(), C.c_size_t()
        check(lib.yb_net_bn_exchange_buffer(self.handle, int(i), int(bool(backward)), C.byref(p), C.byref(n)),
              "yb_net_bn_exchange_buffer")
        off = p.value - self.act.data_ptr()
        return self.act[off: off + n.value * 4].view(torch.float32)

    def bn_batch_stats(self, i):
        """BN layer i's coefficients from the last training forward (include/yolob200.h: yb_net_bn_batch_stats):
        dict(mean, invstd, scale, shift) of float32 [cout] views into the activation arena."""
        ps = [C.c_void_p() for _ in range(4)]
        check(lib.yb_net_bn_batch_stats(self.handle, int(i), *[C.byref(q) for q in ps]), "yb_net_bn_batch_stats")
        c = self.layer_info(i).cout
        out = {}
        for name, q in zip(("mean", "invstd", "scale", "shift"), ps):
            off = q.value - self.act.data_ptr()
            out[name] = self.act[off: off + c * 4].view(torch.float32)
        return out

    def opt_norms(self):
        """Per-tensor squared norms of the last update, float32 [222] view (include/yolob200.h: yb_net_opt_norms)."""
        p, n = C.c_void_p(), C.c_int()
        check(lib.yb_net_opt_norms(self.handle, C.byref(p), C.byref(n)), "yb_net_opt_norms")
        return self._view(p.value, (n.value,))

    def grad_flat(self):
        p, n = C.c_void_p(), C.c_size_t()
        check(lib.yb_net_grad_buffer(self.handle, C.byref(p), C.byref(n)), "yb_net_grad_buffer")
        return self._view(p.value, (n.value,))

    def layer_info(self, i):
        info = _lib.LayerInfo()
        check(lib.yb_net_layer_info(self.handle, i, C.byref(info)), "yb_net_layer_info")
        return info

    def layer_output(self, i):
        """Arena view of one layer's output activation ([n,h,w,ld-strided] -> [n,h,w,cout])."""
        p, ld, dt = C.c_void_p(), C.c_int(), C.c_int()
        check(lib.yb_net_layer_output(self.handle, i, C.byref(p), C.byref(ld), C.byref(dt)), "yb_net_layer_output")
        info = self.layer_info(i)
        tdt = {0: torch.float16, 1: torch.bfloat16, 2: torch.float32, 3: torch.float8_e4m3fn}[dt.value]
        esz = {2: 4, 3: 1}.get(dt.value, 2)
        off = p.value - self.act.data_ptr()
        up = 2 if info.upsample2x else 1
        oh, ow = info.out_h * up, info.out_w * up
        nelem = ((self.n * oh * ow - 1) * ld.value + info.cout)
        flat = self.act[off: off + nelem * esz].view(tdt)
        return flat.as_strided((self.n, oh, ow, info.cout), (oh * ow * ld.value, ow * ld.value, ld.value, 1))

    def fp8_scales(self):
        """e4m3 plan: ([(s_in, s_res, s_out)] per layer, [weight scales float32 [cout_pad] | None] per layer)."""
        act, wts = [], []
        for i in range(self.num_layers):
            v, wp = (C.c_float * 3)(), C.c_void_p()
            check(lib.yb_net_fp8_layer_scales(self.handle, i, v, C.byref(wp)), "yb_net_fp8_layer_scales")
            act.append(tuple(float(a) for a in v))
            wts.append(None if not wp.value else self._view(wp.value, (lib.yb_conv_cout_pad(self.layer_info(i).cout),)).clone())
        return act, wts

    def __del__(self):
        try:
            if self.handle:
                lib.yb_net_destroy(self.handle)
        except Exception:
            pass


class yolov3(object):

    def __init__(self, class_num, anchors, use_label_smooth=False, use_focal_loss=False, batch_norm_decay=0.999,
                 weight_decay=5e-4, use_static_shape=True, dtype="fp16", device=None):
        # model.py:14-28 (same meaning); `dtype`/`device` are engine additions.
        self.class_num = int(class_num)
        self.anchors = np.asarray(anchors, dtype=np.float32).reshape(-1, 2)
        if self.anchors.shape != (9, 2):
            raise ValueError(f"anchors must be [9,2] (w,h) pixels, got {self.anchors.shape}")
        self.batch_norm_decay = batch_norm_decay
        self.use_label_smooth = use_label_smooth
        self.use_focal_loss = use_focal_loss
        self.weight_decay = weight_decay
        self.use_static_shape = use_static_shape
        self._dtype_code, self._torch_dtype = _dtype_code(dtype)
        if not torch.cuda.is_available():
            raise _lib.YoloB200Error("yolov3_tensorflow_b200 needs a CUDA device (sm_100a); there is no CPU fallback")
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.img_size = None
        self._plans = {}
        self._pending = None         # user-supplied parameters not yet uploaded into the arena (75 dicts of CUDA tensors)
        self._pending_layout = _lib.YB_W_HWIO
        self._arena = None           # THE parameter arena (uint8 CUDA tensor), shared by every plan of this model
        self._arena_training = False
        self._have_params = False
        self._fold_dirty = False     # BN parameters / moving statistics changed since the inference scale/shift were folded
        self._opt_kind = None        # optimizer whose slots the arena currently holds
        self._frozen = set()         # conv indices excluded from the update (train.py:81 update_part)
        self.loss_scale = 1024.0 if self._torch_dtype == torch.float16 else 1.0   # static loss scale of the 16-bit backward
        self._fp8_amax = None        # quantize_fp8() models: per-layer calibration amax (their plans are e4m3)

    # ------------------------------------------------------------------ parameters
    @staticmethod
    def conv_table(class_num=80):
        """(cin, cout, ksize, stride, has_bn) of the 75 convs in creation order
        (== TF variable order == darknet .weights order; SURVEY.md Appendix A)."""
        t = []
        c = 3

        def conv(co, k, s=1, bn=True):
            nonlocal c
            t.append((c, co, k, s, bn))
            c = co

        conv(32, 3); conv(64, 3, 2)
        for reps, f in ((1, 32), (2, 64), (8, 128), (8, 256), (4, 512)):
            for _ in range(reps):
                conv(f, 1); conv(2 * f, 3)
            if f != 512:
                conv(4 * f, 3, 2)
        D = 3 * (5 + class_num)
        for cin, f in ((1024, 512), (768, 256), (384, 128)):
            c = cin
            for _ in range(3):
                conv(f, 1); conv(2 * f, 3)
            conv(D, 1, 1, False)
            if f != 128:
                c = f
                conv(f // 2, 1)
        return t

    def _not_fp8(self, what):
        if self._fp8_amax is not None:
            raise ValueError(f"{what}: this model is fp8-quantized (inference only, calibrated activation scales); "
                             "change the fp16/bf16 source model and call quantize_fp8() again")

    def set_params(self, params, layout="HWIO"):
        """params: 75 dicts in creation order with 'w' (+ 'gamma','beta','mean','var' | 'b'),
        numpy or torch float32.  layout of 'w': 'HWIO' (TF variables) or 'OIHW' (darknet)."""
        self._not_fp8("set_params")
        self._set_params(params, layout)

    def _set_params(self, params, layout):
        table = self.conv_table(self.class_num)
        if len(params) != len(table):
            raise ValueError(f"expected {len(table)} conv parameter sets, got {len(params)}")
        out = []
        for i, (p, (cin, cout, k, s, bn)) in enumerate(zip(params, table)):
            q = {}
            want = (k, k, cin, cout) if layout == "HWIO" else (cout, cin, k, k)
            for name, v in p.items():
                tv = torch.as_tensor(np.ascontiguousarray(v) if isinstance(v, np.ndarray) else v, dtype=torch.float32)
                q[name] = tv.to(self.device).contiguous()
            if tuple(q["w"].shape) != want:
                raise ValueError(f"conv {i}: weight shape {tuple(q['w'].shape)} != {want}")   # tf.assign validate_shape
            need = ("gamma", "beta", "mean", "var") if bn else ("b",)
            for name in need:
                if name not in q or q[name].numel() != cout:
                    raise ValueError(f"conv {i}: missing/ill-shaped '{name}'")
            out.append(q)
        self._pending = out
        self._pending_layout = _lib.YB_W_HWIO if layout == "HWIO" else _lib.YB_W_OIHW
        self.__dict__.pop("_graphs", None)           # captured graphs bake nothing parameter-dependent, but re-capture anyway

    def init_params(self, seed=0):
        """Random init as the reference graph would (SURVEY.md B.1): Glorot-uniform conv weights,
        gamma=1, beta=0, moving mean 0 / variance 1, zero detection biases (model.py:55-57)."""
        self._not_fp8("init_params")
        rng = np.random.default_rng(seed)
        ps = []
        for cin, cout, k, s, bn in self.conv_table(self.class_num):
            lim = math.sqrt(6.0 / (k * k * (cin + cout)))
            p = {"w": rng.uniform(-lim, lim, (k, k, cin, cout)).astype(np.float32)}
            if bn:
                p.update(gamma=np.ones(cout, np.float32), beta=np.zeros(cout, np.float32),
                         mean=np.zeros(cout, np.float32), var=np.ones(cout, np.float32))
            else:
                p["b"] = np.zeros(cout, np.float32)
            ps.append(p)
        self.set_params(ps, "HWIO")

    def _ensure_arena(self, plan):
        """Make sure the shared parameter arena exists and is large enough for `plan` (a training plan's layout is the
        inference layout plus gradient / optimizer slots / dgrad weights appended), then bind the plan to it."""
        need = max(plan.param_bytes, 256)
        if self._arena is None or self._arena.numel() < need:
            new = torch.zeros(need, dtype=torch.uint8, device=self.device)
            if self._arena is not None:
                new[: self._arena.numel()].copy_(self._arena)          # weights / BN state keep their offsets
            self._arena = new
            for other in self._plans.values():                         # tensor maps hold arena pointers: rebind
                other.bind(self._arena)
        plan.bind(self._arena)
        if plan.training and not self._arena_training:
            self._arena_training = True
            self._opt_kind = None
            if self._have_params:                                      # weights were uploaded through an inference plan
                check(lib.yb_net_train_refresh_dgrad(plan.handle, stream_handle()), "yb_net_train_refresh_dgrad")
        if plan.training:
            for i in self._frozen:
                check(lib.yb_net_set_trainable(plan.handle, i, 0, stream_handle()), "yb_net_set_trainable")

    def _any_plan(self):
        for pl in self._plans.values():
            if not self._arena_training or pl.training:
                return pl
        return None

    def _plan(self, n, h, w, training=False):
        key = (n, h, w)
        plan = self._plans.get(key)
        if plan is not None and training and not plan.training:
            del self._plans[key]                         # upgrade an inference plan to a training plan
            plan = None
        if plan is None:
            plan = _Plan(self, n, h, w, training)
            self._ensure_arena(plan)
            self._plans[key] = plan
        if self._pending is not None:
            st = stream_handle()
            up = plan if (plan.training or not self._arena_training) else self._any_plan()
            for i, q in enumerate(self._pending):
                check(lib.yb_net_set_conv_params(up.handle, i, ptr(q["w"]), self._pending_layout, ptr(q.get("gamma")),
                                                 ptr(q.get("beta")), ptr(q.get("mean")), ptr(q.get("var")),
                                                 ptr(q.get("b")), st), f"yb_net_set_conv_params[{i}]")
            torch.cuda.current_stream().synchronize()    # the staging tensors are released below
            self._pending = None
            self._have_params = True
            self._fold_dirty = False
        if not self._have_params:
            raise _lib.YoloB200Error("no parameters: call load_weights(model, file), set_params() or init_params()")
        if self._fp8_amax is not None and not getattr(plan, "_fp8_set", False):
            # every plan of a quantized model (any batch / resolution) uses the one calibrated set of scales
            a = self._fp8_amax
            check(lib.yb_net_set_fp8_amax(plan.handle, (C.c_float * len(a))(*a), len(a), stream_handle()), "yb_net_set_fp8_amax")
            plan._fp8_set = True
        return plan

    # ------------------------------------------------------------------ calibrated fp8 (e4m3) inference
    def quantize_fp8(self, calib_images):
        """-> a new inference-only model that runs the convs after Conv_3 with e4m3 activations and weights.

        calib_images: one float32 [N,H,W,3] batch or a list of them.  This model's inference forward runs on each; the
        max |x| of every layer output over all batches (yb_amax) sets the per-buffer activation scales
        (amax / 448, buffers with two producers take the larger), and the weights are quantized per output channel
        from this model's float32 master parameters.  This model is left as it was.  The quantized model supports
        forward(is_training=False), predict, predict_scores, detect_raw, detect and detect_graphed at any batch size
        and resolution; training and parameter changes raise ValueError."""
        self._not_fp8("quantize_fp8")
        batches = calib_images if isinstance(calib_images, (list, tuple)) else [calib_images]
        if not batches:
            raise ValueError("quantize_fp8: no calibration images")
        amax = None
        out = torch.empty(1, dtype=torch.float32, device=self.device)
        for xb in batches:
            self.forward(xb)
            plan = self._last_plan
            vals = torch.zeros(plan.num_layers, dtype=torch.float32, device=self.device)
            for i in range(1, plan.num_layers):      # layer 0's output is never written (the stem is fused into Conv_1)
                if not plan.layer_info(i).has_bn:
                    continue                         # detection heads: float32 outputs, no scale
                y = plan.layer_output(i)
                p, ld, dt = C.c_void_p(), C.c_int(), C.c_int()
                check(lib.yb_net_layer_output(plan.handle, i, C.byref(p), C.byref(ld), C.byref(dt)), "yb_net_layer_output")
                rows = y.shape[0] * y.shape[1] * y.shape[2]
                check(lib.yb_amax(p, ld.value, rows, y.shape[3], dt.value, ptr(out), stream_handle()), "yb_amax")
                vals[i] = out[0]
            amax = vals if amax is None else torch.maximum(amax, vals)
        q = yolov3(self.class_num, self.anchors, self.use_label_smooth, self.use_focal_loss, self.batch_norm_decay,
                   self.weight_decay, self.use_static_shape, dtype="fp16", device=self.device)
        q._dtype_code = _lib.YB_E4M3
        q._set_params(self.get_params(), "HWIO")
        q._fp8_amax = [float(v) for v in amax.cpu().tolist()]
        return q

    def fp8_scales(self):
        """quantize_fp8() models: dict(act=[(s_in, s_res, s_out)] per layer: the scales of the layer's input, residual
        and output buffers (1 for fp16 / float32 buffers), weight=[float32 CPU tensor [cout_pad] | None] per layer:
        the per-output-channel weight scales (None for the fp16 layers 0-3))."""
        if self._fp8_amax is None:
            raise ValueError("fp8_scales: not an fp8-quantized model (see quantize_fp8)")
        plan = self._last_plan if getattr(self, "_last_plan", None) is not None else next(iter(self._plans.values()), None)
        if plan is None:
            raise _lib.YoloB200Error("fp8_scales: run the model once first (its scales are set when a plan is built)")
        act, wts = plan.fp8_scales()
        return {"act": act, "weight": [None if w is None else w.cpu() for w in wts]}

    def set_trainable(self, conv_indices, trainable=True):
        """train.py:81 `update_part`: conv indices (creation order, 0..74) whose weights / BN affine / bias the
        optimizer updates (True) or leaves untouched (False).  The default trains all 222 tensors."""
        for i in conv_indices:
            if trainable:
                self._frozen.discard(int(i))
            else:
                self._frozen.add(int(i))
        for pl in self._plans.values():
            if pl.training:
                for i in conv_indices:
                    check(lib.yb_net_set_trainable(pl.handle, int(i), int(bool(trainable)), stream_handle()), "yb_net_set_trainable")
                break        # the table lives in the shared arena: one upload serves every plan

    # ------------------------------------------------------------------ model.py:30-80
    def forward(self, inputs, is_training=False, reuse=False):
        """inputs float32 [N,H,W,3] in [0,1] (RGB) -> (feature_map_1, feature_map_2, feature_map_3),
        float32 NHWC [N,H/32,W/32,3*(5+C)], [N,H/16,...], [N,H/8,...].  Sets self.img_size (model.py:33)."""
        x = _as_cuda_f32(inputs, self.device)
        if x.dim() != 4 or x.shape[3] != 3:
            raise ValueError(f"inputs must be [N,H,W,3], got {tuple(x.shape)}")
        n, h, w = int(x.shape[0]), int(x.shape[1]), int(x.shape[2])
        if h % 32 or w % 32:
            raise ValueError(f"H and W must be multiples of 32, got {h}x{w}")
        self.img_size = (h, w)
        if is_training:
            self._not_fp8("forward(is_training=True)")
        plan = self._plan(n, h, w, training=bool(is_training))
        D = 3 * (5 + self.class_num)
        fms = [torch.empty((n, h // s, w // s, D), dtype=torch.float32, device=self.device) for s in (32, 16, 8)]
        if is_training:
            # BN uses batch statistics and the moving statistics are updated (UPDATE_OPS, train.py:108-109)
            check(lib.yb_net_train_fwd_bwd(plan.handle, ptr(x), None, None, None, None, 0, 0, float(self.batch_norm_decay),
                                           1.0, ptr(fms[0]), ptr(fms[1]), ptr(fms[2]), None, 1, stream_handle()),
                  "yb_net_train_fwd_bwd(forward_only)")
            self._fold_dirty = True                      # moving statistics changed
        else:
            if self._fold_dirty:                         # another plan trained on the shared arena: refold BN
                check(lib.yb_net_refold_bn(plan.handle, stream_handle()), "yb_net_refold_bn")
                self._fold_dirty = False
            check(lib.yb_net_forward(plan.handle, ptr(x), ptr(fms[0]), ptr(fms[1]), ptr(fms[2]), stream_handle()),
                  "yb_net_forward")
        self._last_plan = plan
        return fms[0], fms[1], fms[2]

    # ------------------------------------------------------------------ model.py:82-137
    def reorg_layer(self, feature_map, anchors):
        if self.img_size is None:
            raise _lib.YoloB200Error("reorg_layer: call forward() first (it records img_size, model.py:33)")
        fm = _as_cuda_f32(feature_map, self.device)
        anchors = np.asarray(anchors, np.float32).reshape(3, 2)
        n, gh, gw, d = fm.shape
        C_ = self.class_num
        if d != 3 * (5 + C_):
            raise ValueError(f"feature_map last dim {d} != 3*(5+{C_})")
        dev = self.device
        xy = torch.empty((gh, gw, 1, 2), dtype=torch.float32, device=dev)
        boxes = torch.empty((n, gh, gw, 3, 4), dtype=torch.float32, device=dev)
        conf = torch.empty((n, gh, gw, 3, 1), dtype=torch.float32, device=dev)
        prob = torch.empty((n, gh, gw, 3, C_), dtype=torch.float32, device=dev)
        check(lib.yb_reorg_layer(ptr(fm), n, gh, gw, self.img_size[0], self.img_size[1], C_,
                                 _lib.fptr(anchors.reshape(-1)), ptr(xy), ptr(boxes), ptr(conf), ptr(prob),
                                 stream_handle()), "yb_reorg_layer")
        return xy, boxes, conf, prob

    # ------------------------------------------------------------------ model.py:140-190
    def predict(self, feature_maps, return_scores=False):
        """-> boxes [N,B,4] (xmin,ymin,xmax,ymax), confs [N,B,1], probs [N,B,C]
        (+ scores = confs*probs, the caller-side op of test_single_image.py:55, if return_scores)."""
        if self.img_size is None:
            raise _lib.YoloB200Error("predict: call forward() first (it records img_size, model.py:33)")
        fms = [_as_cuda_f32(f, self.device) for f in feature_maps]
        if len(fms) != 3:
            raise ValueError("predict expects 3 feature maps")
        n = fms[0].shape[0]
        h, w = self.img_size
        C_ = self.class_num
        for f, s in zip(fms, (32, 16, 8)):
            if tuple(f.shape) != (n, h // s, w // s, 3 * (5 + C_)):
                raise ValueError(f"feature map shape {tuple(f.shape)} does not match img_size {self.img_size}")
        B = 3 * sum((h // s) * (w // s) for s in (32, 16, 8))
        dev = self.device
        boxes = torch.empty((n, B, 4), dtype=torch.float32, device=dev)
        confs = torch.empty((n, B, 1), dtype=torch.float32, device=dev)
        probs = torch.empty((n, B, C_), dtype=torch.float32, device=dev)
        scores = torch.empty((n, B, C_), dtype=torch.float32, device=dev) if return_scores else None
        check(lib.yb_predict(ptr(fms[0]), ptr(fms[1]), ptr(fms[2]), n, h, w, C_, _lib.fptr(self.anchors.reshape(-1)),
                             ptr(boxes), ptr(confs), ptr(probs), ptr(scores), stream_handle()), "yb_predict")
        if return_scores:
            return boxes, confs, probs, scores
        return boxes, confs, probs

    def predict_scores(self, feature_maps):
        """Detection-pipeline variant of predict(): only what gpu_nms consumes — boxes [N,B,4] and
        scores = confs*probs [N,B,C] (test_single_image.py:53-55 fused into one pass, nothing else written)."""
        if self.img_size is None:
            raise _lib.YoloB200Error("predict_scores: call forward() first (it records img_size, model.py:33)")
        fms = [_as_cuda_f32(f, self.device) for f in feature_maps]
        n = fms[0].shape[0]
        h, w = self.img_size
        C_ = self.class_num
        B = 3 * sum((h // s) * (w // s) for s in (32, 16, 8))
        boxes = torch.empty((n, B, 4), dtype=torch.float32, device=self.device)
        scores = torch.empty((n, B, C_), dtype=torch.float32, device=self.device)
        check(lib.yb_predict(ptr(fms[0]), ptr(fms[1]), ptr(fms[2]), n, h, w, C_, _lib.fptr(self.anchors.reshape(-1)),
                             ptr(boxes), None, None, ptr(scores), stream_handle()), "yb_predict")
        return boxes, scores

    # ------------------------------------------------------------------ test_single_image.py:50-57
    def detect_raw(self, inputs, max_boxes=200, score_thresh=0.3, nms_thresh=0.45, phases=7, out=None):
        """The detection pipeline of test_single_image.py:50-57 for a batch, in ONE engine call:
        forward -> predict -> pred_scores = confs * probs -> gpu_nms per image.  The anchor decode and the score filter
        run inside the detection-head conv epilogues (no feature map / score tensor round trip through HBM); results
        are bit-identical to forward() + predict_scores() + batched_nms_raw().
        -> (boxes_all [N,B,4], out_boxes [N,C*max_boxes,4], out_scores, out_labels, out_indices [N,C*max_boxes],
            counts [N]) on the device, no host synchronisation.
        phases / out: benchmarks bracket the parts (1 stem, 2 tensor-core convs, 4 NMS) with their own events and pass
        the previous call's result tuple back in as `out`.
        The fused heads cover 1 to 80 classes, in every dtype and on quantize_fp8 models.  A model with more classes
        runs the three calls instead (same results; phases and out are then ignored)."""
        x = _as_cuda_f32(inputs, self.device)
        if x.dim() != 4 or x.shape[3] != 3:
            raise ValueError(f"inputs must be [N,H,W,3], got {tuple(x.shape)}")
        n, h, w = int(x.shape[0]), int(x.shape[1]), int(x.shape[2])
        if h % 32 or w % 32:
            raise ValueError(f"H and W must be multiples of 32, got {h}x{w}")
        self.img_size = (h, w)
        plan = self._plan(n, h, w, training=False)
        if self._fold_dirty:
            check(lib.yb_net_refold_bn(plan.handle, stream_handle()), "yb_net_refold_bn")
            self._fold_dirty = False
        self._last_plan = plan
        C_, mb = self.class_num, int(max_boxes)
        if not lib.yb_net_detect_supported(plan.handle):
            from .utils.nms_utils import batched_nms_raw       # class counts without a fused kernel: three calls
            boxes, scores = self.predict_scores(self.forward(x))
            return (boxes,) + tuple(batched_nms_raw(boxes, scores, C_, mb, score_thresh, nms_thresh))
        B = 3 * sum((h // s) * (w // s) for s in (32, 16, 8))
        dev = self.device
        cap = max(C_ * max(mb, 0), 1)
        if out is not None:
            boxes, ob, os_, ol, oi, cnt = out
        else:
            boxes = torch.empty((n, B, 4), dtype=torch.float32, device=dev)
            ob = torch.empty((n, cap, 4), dtype=torch.float32, device=dev)
            os_ = torch.empty((n, cap), dtype=torch.float32, device=dev)
            ol = torch.empty((n, cap), dtype=torch.int32, device=dev)
            oi = torch.empty((n, cap), dtype=torch.int32, device=dev)
            cnt = torch.empty((n,), dtype=torch.int32, device=dev)
        need = C.c_size_t()
        check(lib.yb_net_detect_workspace_bytes(plan.handle, mb, C.byref(need)), "yb_net_detect_workspace_bytes")
        ws = getattr(plan, "_det_ws", None)
        if ws is None or ws.numel() < need.value:
            ws = torch.empty(max(need.value, 256), dtype=torch.uint8, device=dev)
            plan._det_ws = ws                                  # per plan: stream-ordered reuse by this model only
        check(lib.yb_net_detect_phases(plan.handle, ptr(x), _lib.fptr(self.anchors.reshape(-1)), mb, float(score_thresh),
                                       float(nms_thresh), ptr(ws), ws.numel(), ptr(boxes), ptr(ob), ptr(os_), ptr(ol),
                                       ptr(oi), ptr(cnt), int(phases), stream_handle()), "yb_net_detect")
        return boxes, ob, os_, ol, oi, cnt

    def detect_graphed(self, inputs, max_boxes=200, score_thresh=0.3, nms_thresh=0.45):
        """detect_raw() replayed from a CUDA graph (SURVEY.md 7 step 6): the 76 launches of a detection step are captured
        once per (input shape, thresholds) and replayed with one cudaGraphLaunch — for the single-image path of
        test_single_image.py:48-62, where launch overhead, not the kernels, is the latency.  The input is copied into the
        graph's static buffer; the returned tensors are the graph's static outputs (overwritten by the next call)."""
        x = _as_cuda_f32(inputs, self.device)
        key = (tuple(x.shape), int(max_boxes), float(score_thresh), float(nms_thresh))
        graphs = self.__dict__.setdefault("_graphs", {})
        entry = graphs.get(key)
        if entry is None or self._fold_dirty or self._pending is not None:
            sx = x.clone()
            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream()
            side.wait_stream(cur)
            with torch.cuda.stream(side):                 # warm-up outside the capture: plan, kernel attributes, workspace
                for _ in range(2):
                    self.detect_raw(sx, max_boxes, score_thresh, nms_thresh)
            cur.wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = self.detect_raw(sx, max_boxes, score_thresh, nms_thresh)
            entry = graphs[key] = (g, sx, out)
        g, sx, out = entry
        sx.copy_(x, non_blocking=True)
        g.replay()
        return out

    def detect(self, inputs, max_boxes=200, score_thresh=0.3, nms_thresh=0.45):
        """detect_raw() unpacked like the reference's per-image result: a list of (boxes [K,4], scores [K], labels [K])
        per image (classes ascending, descending score inside a class).  Reading the counts is the one host sync."""
        _, ob, os_, ol, oi, cnt = self.detect_raw(inputs, max_boxes, score_thresh, nms_thresh)
        return [(ob[i, :k], os_[i, :k], ol[i, :k]) for i, k in enumerate(cnt.tolist())]

    # ------------------------------------------------------------------ model.py:192-304
    def _loss_scale(self, feature_map_i, y_true, anchors, loss4, want_grad=False, grad_out=None):
        fm = _as_cuda_f32(feature_map_i, self.device)
        yt = _as_cuda_f32(y_true, self.device)
        n, gh, gw, d = fm.shape
        C_ = self.class_num
        if d != 3 * (5 + C_):
            raise ValueError(f"feature_map last dim {d} != 3*(5+{C_})")
        if tuple(yt.shape) != (n, gh, gw, 3, 6 + C_):
            raise ValueError(f"y_true shape {tuple(yt.shape)} != {(n, gh, gw, 3, 6 + C_)}")
        if self.img_size is None:
            raise _lib.YoloB200Error("loss_layer: call forward() first (it records img_size, model.py:33)")
        need = C.c_size_t()
        check(lib.yb_loss_workspace_bytes(n, gh, gw, C.byref(need)), "yb_loss_workspace_bytes")
        ws = torch.empty(need.value, dtype=torch.uint8, device=self.device)
        grad = None
        if want_grad:
            grad = grad_out if grad_out is not None else torch.empty_like(fm)
        anchors = np.asarray(anchors, np.float32).reshape(3, 2)
        check(lib.yb_loss_layer(ptr(fm), ptr(yt), n, gh, gw, self.img_size[0], self.img_size[1], C_,
                                _lib.fptr(anchors.reshape(-1)), int(self.use_label_smooth), int(self.use_focal_loss),
                                1.0 / n, 1.0, ptr(ws), ws.numel(), ptr(loss4), ptr(grad), _lib.YB_F32, 0, stream_handle()),
              "yb_loss_layer")
        return grad

    def loss_layer(self, feature_map_i, y_true, anchors):
        """model.py:192-304 -> (xy_loss, wh_loss, conf_loss, class_loss), 0-dim float32 CUDA tensors."""
        l4 = torch.zeros(4, dtype=torch.float64, device=self.device)
        self._loss_scale(feature_map_i, y_true, anchors, l4)
        out = torch.empty(5, dtype=torch.float32, device=self.device)
        check(lib.yb_loss_finalize(ptr(l4), ptr(out), stream_handle()), "yb_loss_finalize")
        return out[1], out[2], out[3], out[4]

    def box_iou(self, pred_boxes, valid_true_boxes):
        """model.py:307-345: pred_boxes [g,g,3,4], valid_true_boxes [V,4] (cx,cy,w,h) -> [g,g,3,V]."""
        pb = _as_cuda_f32(pred_boxes, self.device)
        tb = _as_cuda_f32(valid_true_boxes, self.device).reshape(-1, 4)
        lead = tuple(pb.shape[:-1])
        P, V = int(np.prod(lead)), tb.shape[0]
        out = torch.empty(lead + (V,), dtype=torch.float32, device=self.device)
        check(lib.yb_box_iou(ptr(pb), ptr(tb), P, V, ptr(out), stream_handle()), "yb_box_iou")
        return out

    def compute_loss(self, y_pred, y_true, return_grads=False):
        """model.py:348-365 -> [total_loss, loss_xy, loss_wh, loss_conf, loss_class] (0-dim float32 CUDA
        tensors).  return_grads=True additionally returns d(total)/d(feature_map_i) for the three scales
        (what train.py:112's compute_gradients back-propagates into the network)."""
        if len(y_pred) != 3 or len(y_true) != 3:
            raise ValueError("compute_loss expects 3 feature maps and 3 y_true tensors")
        groups = [self.anchors[6:9], self.anchors[3:6], self.anchors[0:3]]
        l4 = torch.zeros(4, dtype=torch.float64, device=self.device)
        grads = [self._loss_scale(y_pred[i], y_true[i], groups[i], l4, want_grad=return_grads) for i in range(3)]
        out = torch.empty(5, dtype=torch.float32, device=self.device)
        check(lib.yb_loss_finalize(ptr(l4), ptr(out), stream_handle()), "yb_loss_finalize")
        losses = [out[0], out[1], out[2], out[3], out[4]]
        return (losses, grads) if return_grads else losses

    # ------------------------------------------------------------------ train.py:105-115
    def get_params(self):
        """Current parameters as 75 dicts of numpy arrays, weights in TF's HWIO layout."""
        if self._pending is not None:
            out = []
            for q in self._pending:
                d = {k: v.detach().cpu().numpy() for k, v in q.items()}
                if self._pending_layout == _lib.YB_W_OIHW:
                    d["w"] = np.ascontiguousarray(np.transpose(d["w"], (2, 3, 1, 0)))
                elif self._pending_layout == _lib.YB_W_OHWI:
                    d["w"] = np.ascontiguousarray(np.transpose(d["w"], (1, 2, 3, 0)))
                out.append(d)
            return out
        plan = self._any_plan()
        if plan is None or not self._have_params:
            raise _lib.YoloB200Error("no parameters")
        out = []
        for i in range(plan.num_layers):
            d = {k: v.detach().cpu().numpy() for k, v in plan.conv_params(i).items()}
            d["w"] = np.ascontiguousarray(np.transpose(d["w"], (1, 2, 3, 0)))      # arena OHWI -> HWIO
            out.append(d)
        return out

    def optimizer_state(self):
        """(slots [num_slots, count] float32 view, ctrl int32[3] view = [non-finite flag, updates applied, steps skipped])
        of the shared optimizer state — what `save_optimizer=True` (args.py:37, train.py:101-104) checkpoints."""
        plan = next((pl for pl in self._plans.values() if pl.training), None)
        if plan is None:
            raise _lib.YoloB200Error("optimizer_state: no training plan yet")
        sl, cnt, ns, ctrl = C.c_void_p(), C.c_size_t(), C.c_int(), C.c_void_p()
        check(lib.yb_net_opt_state(plan.handle, C.byref(sl), C.byref(cnt), C.byref(ns), C.byref(ctrl)), "yb_net_opt_state")
        off = sl.value - self._arena.data_ptr()
        slots = self._arena[off: off + ns.value * cnt.value * 4].view(torch.float32).view(ns.value, cnt.value)
        coff = ctrl.value - self._arena.data_ptr()
        return slots, self._arena[coff: coff + 12].view(torch.int32)

    def _train_setup(self, images, y_true, learning_rate, momentum, clip_norm, optimizer, decay, beta1, beta2, epsilon,
                     return_feature_maps):
        """Checks and state shared by the training-step entry points -> (x, ys, plan, opt without grad_scale, fms)."""
        x = _as_cuda_f32(images, self.device)
        ys = [_as_cuda_f32(y, self.device) for y in y_true]
        n, h, w = int(x.shape[0]), int(x.shape[1]), int(x.shape[2])
        if h % 32 or w % 32 or x.shape[3] != 3:
            raise ValueError(f"images must be [N,H,W,3] with H,W multiples of 32, got {tuple(x.shape)}")
        C_ = self.class_num
        for y, s in zip(ys, (32, 16, 8)):
            if tuple(y.shape) != (n, h // s, w // s, 3, 6 + C_):
                raise ValueError(f"y_true shape {tuple(y.shape)} != {(n, h // s, w // s, 3, 6 + C_)}")
        if hasattr(optimizer, "name"):                   # utils.misc_utils.config_optimizer(...) object
            momentum, decay = getattr(optimizer, "momentum", momentum), getattr(optimizer, "decay", decay)
            optimizer = optimizer.name
        kinds = {"sgd": _lib.YB_OPT_SGD, "momentum": _lib.YB_OPT_MOMENTUM, "rmsprop": _lib.YB_OPT_RMSPROP, "adam": _lib.YB_OPT_ADAM}
        if optimizer not in kinds:
            raise ValueError("Unsupported optimizer type!")                 # utils/misc_utils.py:161
        kind = kinds[optimizer]
        if epsilon is None:
            epsilon = 1e-10 if kind == _lib.YB_OPT_RMSPROP else 1e-8        # [TF] defaults
        self.img_size = (h, w)
        plan = self._plan(n, h, w, training=True)
        st = stream_handle()
        if self._opt_kind != kind:                                          # fresh arena or optimizer switch: new slots
            check(lib.yb_net_train_reset_state(plan.handle, kind, st), "yb_net_train_reset_state")
            self._opt_kind = kind
            saved = getattr(self, "_restore_optimizer", None)               # utils.misc_utils.restore_checkpoint
            if saved is not None and saved[2] == kind:
                slots, ctrl = self.optimizer_state()
                if tuple(slots.shape) != tuple(saved[0].shape):
                    raise ValueError(f"optimizer slots in the checkpoint have shape {saved[0].shape}, expected {tuple(slots.shape)}")
                slots.copy_(torch.from_numpy(saved[0]).to(self.device))
                ctrl.copy_(torch.from_numpy(saved[1]).to(self.device))
            self._restore_optimizer = None
        fms = [None, None, None]
        if return_feature_maps:
            fms = [torch.empty((n, h // s, w // s, 3 * (5 + C_)), dtype=torch.float32, device=self.device) for s in (32, 16, 8)]
        opt = _lib.Optimizer(kind=kind, lr=float(learning_rate), grad_scale=0.0, momentum=float(momentum),
                             decay=float(decay), beta1=float(beta1), beta2=float(beta2), epsilon=float(epsilon),
                             weight_decay=float(self.weight_decay), clip_norm=float(clip_norm))
        return x, ys, plan, opt, fms

    @staticmethod
    def _grad_buckets(plan, bucket_mb):
        from .parallel import gradient_buckets
        if not hasattr(plan, "_buckets") or plan._bucket_mb != bucket_mb:
            sizes = [plan.grad_range(i, i).numel() for i in range(plan.num_layers)]
            plan._buckets = gradient_buckets(sizes, int(bucket_mb * (1 << 20) / 4))
            plan._bucket_mb = bucket_mb
        return plan._buckets

    def _finish_step(self, plan, opt, grad_scale, fms, return_feature_maps):
        st = stream_handle()
        opt.grad_scale = grad_scale
        check(lib.yb_net_train_update(plan.handle, C.byref(opt), st), "yb_net_train_update")
        self._fold_dirty = True
        self._last_plan = plan
        out = torch.empty(5, dtype=torch.float32, device=self.device)
        check(lib.yb_loss_finalize(ptr(plan.loss4), ptr(out), st), "yb_loss_finalize")
        losses = [out[0], out[1], out[2], out[3], out[4]]
        return (losses, fms) if return_feature_maps else losses

    def train_step(self, images, y_true, learning_rate, momentum=0.9, clip_norm=100.0, process_group=None,
                   return_feature_maps=False, data_parallel=True, optimizer="momentum", decay=0.9, beta1=0.9,
                   beta2=0.999, epsilon=None, freeze_bn=False, bucket_mb=32.0, sync_bn=False):
        """One training step of the reference (train.py:105-115): forward(is_training=True) -> compute_loss ->
        gradients of (loss[0] + l2_loss) w.r.t. the trainable tensors (all 222 unless set_trainable() restricted them,
        train.py:81) -> per-tensor clip_by_norm(clip_norm) -> optimizer update; BN moving statistics updated with
        self.batch_norm_decay.

        images float32 [N,H,W,3]; y_true = (y_true_13, y_true_26, y_true_52) in process_box format.
        learning_rate: this step's value (utils.misc_utils.config_learning_rate / learning_rate_at evaluate the
        reference's schedules on the host).  optimizer: 'momentum' (default), 'sgd', 'rmsprop', 'adam' or the object
        returned by utils.misc_utils.config_optimizer (utils/misc_utils.py:151-161; TF1 update rules).
        freeze_bn: BN layers normalise with their moving statistics and keep them (the graph the reference builds with
        is_training=False, train.py:72): fine-tuning with frozen BN.
        Data parallel: when torch.distributed is initialised (or process_group is given) the flat gradient is
        all-reduced (NCCL over NVLink) and averaged over the ranks before the update; every loss term is a
        mean over the local batch (model.py:276-302), so this equals one big batch of world*N images.  The gradient
        is reduced in buckets of ~bucket_mb MB, detection heads first, each all-reduce overlapping the backward of
        the layers below it (bucket_mb <= 0: one blocking all-reduce after the whole backward).
        sync_bn: synchronised batch norm across the ranks.  Training-mode BN then normalises with the statistics of
        the global batch and back-propagates through them, so the step equals the single-device step on the
        concatenated batch (up to fp32 summation order) and every rank holds the same moving statistics.  Every rank
        must run the same N, H and W.  Runs train_step_sync_bn() over NCCL; with one rank it is the ordinary step.
        Returns [total, xy, wh, conf, class] as 0-dim float32 CUDA tensors of the LOCAL batch."""
        self._not_fp8("train_step")
        import torch.distributed as dist
        if sync_bn and freeze_bn:
            raise ValueError("sync_bn=True needs training-mode BN: frozen BN (freeze_bn=True) has no batch statistics to synchronise")
        from .parallel import allreduce_gradients, BucketedAllReduce
        use_dp = data_parallel and (process_group is not None or (dist.is_available() and dist.is_initialized()))
        use_dp = use_dp and dist.get_world_size(process_group) > 1
        if sync_bn and use_dp:
            gen = self.train_step_sync_bn(images, y_true, learning_rate, dist.get_world_size(process_group), momentum,
                                          clip_norm, return_feature_maps, optimizer, decay, beta1, beta2, epsilon, bucket_mb)
            return _drive_sync_bn(gen, process_group)
        x, ys, plan, opt, fms = self._train_setup(images, y_true, learning_rate, momentum, clip_norm, optimizer, decay,
                                                  beta1, beta2, epsilon, return_feature_maps)
        st = stream_handle()
        flags = _lib.YB_TRAIN_BN_FROZEN if freeze_bn else 0
        bucketed = use_dp and bucket_mb and bucket_mb > 0
        check(lib.yb_net_train_fwd_bwd(plan.handle, ptr(x), ptr(ys[0]), ptr(ys[1]), ptr(ys[2]),
                                       _lib.fptr(self.anchors.reshape(-1)), int(self.use_label_smooth),
                                       int(self.use_focal_loss), float(self.batch_norm_decay), float(self.loss_scale),
                                       ptr(fms[0]), ptr(fms[1]), ptr(fms[2]), ptr(plan.loss4),
                                       flags | (_lib.YB_TRAIN_NO_BACKWARD if bucketed else 0), st), "yb_net_train_fwd_bwd")
        grad_scale = 1.0 / float(self.loss_scale)
        if bucketed:
            # backward bucket by bucket (heads first); each bucket's all-reduce overlaps the next bucket's backward
            red = BucketedAllReduce(process_group)
            for lo, hi in self._grad_buckets(plan, bucket_mb):
                check(lib.yb_net_train_backward(plan.handle, ptr(x), lo, hi, flags, st), "yb_net_train_backward")
                red.reduce(plan.grad_range(lo, hi))
            grad_scale *= red.wait()
        elif use_dp:
            grad_scale *= allreduce_gradients(plan.grad_flat(), process_group)   # NCCL all-reduce (sum) -> 1/world
        return self._finish_step(plan, opt, grad_scale, fms, return_feature_maps)

    def train_step_sync_bn(self, images, y_true, learning_rate, bn_replicas, momentum=0.9, clip_norm=100.0,
                           return_feature_maps=False, optimizer="momentum", decay=0.9, beta1=0.9, beta2=0.999,
                           epsilon=None, bucket_mb=32.0):
        """train_step(sync_bn=True) as a generator that leaves the transport to its caller.

        The step runs layer by layer (include/yolob200.h: yb_net_train_forward_layer).  At every exchange point it
        yields (kind, tensor), and the caller sums the tensor in place across the bn_replicas ranks:
          ("bn", slab)        a BN layer's forward [Σz | Σz²] or backward [Σdact·ẑ | Σdact] sums; the next layer
                              call consumes the sum, so it is on the critical path;
          ("grad", slice)     a finished gradient bucket (heads first; the whole flat gradient when bucket_mb <= 0);
          ("grad_scale", None) after the last bucket: send back the factor that turns the summed gradient into the
                              mean (1/world), which the optimizer folds in.
        Then the update and the loss finalize run as in train_step, and the generator returns what train_step
        returns.  Every rank must run the same number of images and the same H x W."""
        self._not_fp8("train_step_sync_bn")
        bn_replicas = int(bn_replicas)
        if bn_replicas < 1:
            raise ValueError(f"bn_replicas must be >= 1, got {bn_replicas}")
        x, ys, plan, opt, fms = self._train_setup(images, y_true, learning_rate, momentum, clip_norm, optimizer, decay,
                                                  beta1, beta2, epsilon, return_feature_maps)
        st = stream_handle()
        h, L = plan.handle, plan.num_layers
        has_bn = [bool(plan.layer_info(i).has_bn) for i in range(L)]
        decay_bn = float(self.batch_norm_decay)
        for i in range(L):
            check(lib.yb_net_train_forward_layer(h, ptr(x), i, _lib.YB_PHASE_LOCAL, bn_replicas, decay_bn, ptr(fms[0]),
                                                 ptr(fms[1]), ptr(fms[2]), 0, st), "yb_net_train_forward_layer")
            if has_bn[i]:
                yield "bn", plan.bn_exchange_buffer(i, backward=False)
            check(lib.yb_net_train_forward_layer(h, ptr(x), i, _lib.YB_PHASE_GLOBAL, bn_replicas, decay_bn, ptr(fms[0]),
                                                 ptr(fms[1]), ptr(fms[2]), 0, st), "yb_net_train_forward_layer")
        check(lib.yb_net_train_loss(h, ptr(ys[0]), ptr(ys[1]), ptr(ys[2]), _lib.fptr(self.anchors.reshape(-1)),
                                    int(self.use_label_smooth), int(self.use_focal_loss), float(self.loss_scale),
                                    ptr(plan.loss4), st), "yb_net_train_loss")
        bucketed = bucket_mb and bucket_mb > 0
        for lo, hi in (self._grad_buckets(plan, bucket_mb) if bucketed else [(0, L - 1)]):
            for i in range(hi, lo - 1, -1):
                check(lib.yb_net_train_backward_layer(h, ptr(x), i, _lib.YB_PHASE_LOCAL, bn_replicas, 0, st),
                      "yb_net_train_backward_layer")
                if has_bn[i]:
                    yield "bn", plan.bn_exchange_buffer(i, backward=True)
                check(lib.yb_net_train_backward_layer(h, ptr(x), i, _lib.YB_PHASE_GLOBAL, bn_replicas, 0, st),
                      "yb_net_train_backward_layer")
            check(lib.yb_net_train_join(h, st), "yb_net_train_join")
            yield "grad", (plan.grad_range(lo, hi) if bucketed else plan.grad_flat())
        factor = yield "grad_scale", None
        return self._finish_step(plan, opt, float(factor) / float(self.loss_scale), fms, return_feature_maps)


def _drive_sync_bn(gen, group):
    """Run a train_step_sync_bn generator over torch.distributed: BN slabs are summed on their own communicator
    (parallel.sync_bn_group), gradient buckets by BucketedAllReduce on `group`."""
    import torch.distributed as dist
    from .parallel import BucketedAllReduce, sync_bn_group
    bn_group = sync_bn_group(group)
    red = BucketedAllReduce(group)
    reply = None
    try:
        while True:
            kind, t = gen.send(reply)
            reply = None
            if kind == "bn":
                dist.all_reduce(t, op=dist.ReduceOp.SUM, group=bn_group)
            elif kind == "grad":
                red.reduce(t)
            else:
                reply = red.wait()
    except StopIteration as done:
        return done.value
