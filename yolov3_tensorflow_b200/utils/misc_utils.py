"""The hot-path subset of the reference's utils/misc_utils.py: anchor / class-name parsers, the darknet
`.weights` loader (utils/misc_utils.py:31-47, 70-126), the learning-rate schedules and optimizer selection
(:129-161) and the checkpoint naming of convert_weight.py / train.py."""
from __future__ import annotations

import os

import numpy as np


def parse_anchors(anchor_path):
    """utils/misc_utils.py:31-37 -> float32 [N,2] (w,h)."""
    with open(anchor_path, "r") as f:
        return np.reshape(np.asarray(f.readline().split(","), np.float32), [-1, 2])


def read_class_names(class_name_path):
    """utils/misc_utils.py:40-45 -> {id: name}."""
    names = {}
    with open(class_name_path, "r") as data:
        for i, name in enumerate(data):
            names[i] = name.strip("\n")
    return names


DEFAULT_ANCHOR_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "data", "yolo_anchors.txt")
DEFAULT_CLASS_NAME_PATH = os.path.join(os.path.dirname(DEFAULT_ANCHOR_PATH), "coco.names")


def load_weights(model, weights_file):
    """utils/misc_utils.py:70-126.  The reference takes the TF variable list; here the first argument
    is the `yolov3` model, whose conv table *is* that creation order.  Stream: 5 x int32 header, then per
    conv [beta, gamma, mean, var] (or [bias]) followed by the weights as (Cout, Cin, kh, kw) float32.
    The (Cout,Cin,kh,kw) -> engine-layout transposition the reference does on the host (:117-120)
    happens on the GPU (yb_pack_conv_weights).  Raises ValueError on a size mismatch
    (tf.assign(validate_shape=True)), and on an fp8-quantized model (yolov3.quantize_fp8), whose weights are fixed."""
    if getattr(model, "_fp8_amax", None) is not None:
        model._not_fp8("load_weights")
    with open(weights_file, "rb") as fp:
        np.fromfile(fp, dtype=np.int32, count=5)
        weights = np.fromfile(fp, dtype=np.float32)
    ptr = 0
    params = []
    for cin, cout, k, s, bn in model.conv_table(model.class_num):
        p = {}
        names = ("beta", "gamma", "mean", "var") if bn else ("b",)
        for name in names:
            if ptr + cout > weights.size:
                raise ValueError("darknet weights file is too short for this architecture")
            p[name] = weights[ptr:ptr + cout]
            ptr += cout
        n = cout * cin * k * k
        if ptr + n > weights.size:
            raise ValueError("darknet weights file is too short for this architecture")
        p["w"] = weights[ptr:ptr + n].reshape(cout, cin, k, k)
        ptr += n
        params.append(p)
    if ptr != weights.size:
        raise ValueError(f"darknet weights file has {weights.size} floats, architecture needs {ptr}")
    model.set_params(params, layout="OIHW")
    return ptr


def save_weights(params, weights_file, layout="HWIO"):
    """Inverse of load_weights (SURVEY.md §8f N2): write 75 parameter dicts as a darknet stream."""
    with open(weights_file, "wb") as f:
        np.array([0, 2, 0, 0, 0], np.int32).tofile(f)
        for p in params:
            if "gamma" in p:
                for k in ("beta", "gamma", "mean", "var"):
                    np.asarray(p[k], np.float32).tofile(f)
            else:
                np.asarray(p["b"], np.float32).tofile(f)
            w = np.asarray(p["w"], np.float32)
            if layout == "HWIO":
                w = np.transpose(w, (3, 2, 0, 1))
            np.ascontiguousarray(w).tofile(f)


# ------------------------------------------------------------------------------------------------
# Learning-rate schedules and optimizer selection (utils/misc_utils.py:129-161, train.py:93-99).
# The reference builds TF graph nodes from `global_step`; here the host evaluates the same function
# once per step and hands the float to `yolov3.train_step(learning_rate=...)`.
# ------------------------------------------------------------------------------------------------
def config_learning_rate(args, global_step):
    """utils/misc_utils.py:129-148 evaluated at float `global_step` (warm-up is NOT applied here, as in the
    reference: train.py:93-99 composes it — see `learning_rate_at`).  TensorFlow 1.x semantics:
    exponential_decay(staircase=True) then a lower bound; the reference's own cosine formula;
    cosine_decay_restarts(t_mul=2.0, m_mul=1.0); a constant; piecewise_constant (value i while
    step <= boundaries[i])."""
    step = float(global_step)
    kind = args.lr_type
    lr0 = float(args.learning_rate_init)
    if kind == "fixed":
        return lr0
    if kind == "exponential":
        periods = np.floor(step / float(args.lr_decay_freq))
        return float(max(lr0 * float(args.lr_decay_factor) ** periods, float(args.lr_lower_bound)))
    if kind == "cosine_decay":
        span = (args.total_epoches - float(args.use_warm_up) * args.warm_up_epoch) * args.train_batch_num
        lo = float(args.lr_lower_bound)
        return float(lo + 0.5 * (lr0 - lo) * (1.0 + np.cos(step / span * np.pi)))
    if kind == "cosine_decay_restart":
        done = step / float(args.lr_decay_freq)            # in units of the first period; period k lasts 2**k
        k = np.floor(np.log2(done + 1.0))
        inside = (done - (2.0 ** k - 1.0)) / 2.0 ** k
        return float(lr0 * 0.5 * (1.0 + np.cos(np.pi * inside)))
    if kind == "piecewise":
        bounds, values = list(args.pw_boundaries), list(args.pw_values)
        if len(values) != len(bounds) + 1:
            raise ValueError("The length of boundaries should be 1 less than the length of values")
        return float(values[int(np.searchsorted(np.asarray(bounds, np.float64), step, side="left"))])
    raise ValueError("Unsupported learning rate type!")


def learning_rate_at(args, global_step):
    """train.py:93-99: linear warm-up to learning_rate_init over warm_up_epoch epochs, then the schedule
    of config_learning_rate on (global_step - warm-up steps)."""
    step = float(global_step)
    if getattr(args, "use_warm_up", False):
        warm = float(args.train_batch_num) * float(args.warm_up_epoch)
        if step < warm:
            return float(args.learning_rate_init) * step / warm
        return config_learning_rate(args, step - warm)
    return config_learning_rate(args, step)


class OptimizerConfig(object):
    """What utils/misc_utils.py:151-161 returns, minus the TF object: the name and hyper-parameters that
    `yolov3.train_step(optimizer=...)` hands to the multi-tensor update kernel (csrc/optim.cu)."""

    def __init__(self, name, learning_rate, decay=0.9, momentum=0.9):
        self.name, self.learning_rate, self.decay, self.momentum = name, learning_rate, decay, momentum

    def __repr__(self):
        return f"OptimizerConfig({self.name!r}, lr={self.learning_rate}, decay={self.decay}, momentum={self.momentum})"


def config_optimizer(optimizer_name, learning_rate, decay=0.9, momentum=0.9):
    """utils/misc_utils.py:151-161: 'momentum' | 'rmsprop' | 'adam' | 'sgd'."""
    if optimizer_name not in ("momentum", "rmsprop", "adam", "sgd"):
        raise ValueError("Unsupported optimizer type!")
    return OptimizerConfig(optimizer_name, learning_rate, decay, momentum)


# ------------------------------------------------------------------------------------------------
# Checkpoint naming (convert_weight.py:28-32, train.py:81,101-104,124): the TF variable names of the
# 366 variables in creation order, and an .npz interchange keyed by them (+ optimizer slots).
# ------------------------------------------------------------------------------------------------
def tf_variable_names(class_num=80):
    """[(conv index, key, 'yolov3/<scope>/Conv[_k]/...:0')] in tf.global_variables(scope='yolov3') order:
    per conv `weights`, then `BatchNorm/{gamma,beta,moving_mean,moving_variance}` or `biases`
    (utils/misc_utils.py:84-112 relies on exactly this order)."""
    from ..model import yolov3
    out = []
    body = head = 0
    for i, (cin, cout, k, s, bn) in enumerate(yolov3.conv_table(class_num)):
        in_head = i >= 52
        idx = head if in_head else body
        scope = "yolov3/" + ("yolov3_head" if in_head else "darknet53_body") + "/Conv" + (f"_{idx}" if idx else "")
        if in_head:
            head += 1
        else:
            body += 1
        out.append((i, "w", scope + "/weights:0"))
        if bn:
            for key, nm in (("gamma", "gamma"), ("beta", "beta"), ("mean", "moving_mean"), ("var", "moving_variance")):
                out.append((i, key, f"{scope}/BatchNorm/{nm}:0"))
        else:
            out.append((i, "b", scope + "/biases:0"))
    return out


def save_checkpoint(model, path, global_step=0, save_optimizer=True):
    """train.py:101-104,118-121 `saver_to_save.save`: an .npz keyed by the TF variable names (weights HWIO like the
    TF variables), plus `global_step` and — when save_optimizer (args.py:37) — the optimizer slots."""
    params = model.get_params()
    blob = {name: params[i][key] for i, key, name in tf_variable_names(model.class_num)}
    blob["global_step"] = np.asarray(float(global_step), np.float32)
    if save_optimizer:
        try:
            slots, ctrl = model.optimizer_state()
            blob["optimizer/slots"] = slots.detach().cpu().numpy()
            blob["optimizer/ctrl"] = ctrl.detach().cpu().numpy()
            blob["optimizer/kind"] = np.asarray(-1 if model._opt_kind is None else model._opt_kind, np.int32)
        except Exception:
            pass                                         # no training plan yet: nothing to save
    np.savez(path, **blob)


def restore_checkpoint(model, path, restore_include=None, restore_exclude=None, restore_optimizer=True):
    """train.py:80,124 `saver_to_restore.restore` with get_variables_to_restore(include, exclude) semantics:
    a variable is restored when its name starts with one of `restore_include` (None: all) and with none of
    `restore_exclude`.  Variables not restored keep the model's current values.  Returns global_step."""
    ck = np.load(path)
    if model._pending is None and not model._have_params:
        model.init_params(0)                             # variables exist (initialised) before saver.restore
    params = model.get_params()

    def wanted(name):
        if restore_include is not None and not any(name.startswith(s) for s in restore_include):
            return False
        return not any(name.startswith(s) for s in (restore_exclude or []))

    for i, key, name in tf_variable_names(model.class_num):
        if name in ck.files and wanted(name):
            if ck[name].shape != params[i][key].shape:
                raise ValueError(f"{name}: checkpoint shape {ck[name].shape} != variable shape {params[i][key].shape}")
            params[i][key] = ck[name]
    model.set_params(params, "HWIO")
    if restore_optimizer and "optimizer/slots" in ck.files:
        model._restore_optimizer = (ck["optimizer/slots"], ck["optimizer/ctrl"], int(ck["optimizer/kind"]))
    return float(ck["global_step"]) if "global_step" in ck.files else 0.0
