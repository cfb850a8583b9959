"""ctypes binding of libyolob200.so (the C ABI declared in include/yolob200.h).

The library is the product: there is no Python/PyTorch fallback.  Importing this
module when the shared object is missing raises immediately.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libyolob200.so")

YB_F16, YB_BF16, YB_F32, YB_E4M3 = 0, 1, 2, 3
YB_W_HWIO, YB_W_OIHW, YB_W_OHWI = 0, 1, 2
YB_OPT_SGD, YB_OPT_MOMENTUM, YB_OPT_RMSPROP, YB_OPT_ADAM = 0, 1, 2, 3
YB_TRAIN_FORWARD_ONLY, YB_TRAIN_BN_FROZEN, YB_TRAIN_NO_BACKWARD = 1, 2, 4
YB_PHASE_LOCAL, YB_PHASE_GLOBAL = 0, 1
YB_VOC_MAX_GT = 1024
YB_KMEANS_MAX_K = 32
YB_JPEG_BAD_MARKER, YB_JPEG_BAD_RST, YB_JPEG_BAD_CODE, YB_JPEG_BAD_INDEX, YB_JPEG_TRUNCATED = 1, 2, 4, 8, 16
YB_PLOT_BAD_LABEL, YB_PLOT_BAD_BOX, YB_PLOT_SUFFIX_MAX = 1, 2, 48
YB_JPEG_SAMPLING = {"411": 0x411111, "420": 0x221111, "422": 0x211111, "440": 0x121111, "444": 0x111111}
YB_LAYER_IGEMM, YB_LAYER_HALO, YB_LAYER_FUSED_STEM, YB_LAYER_STEM, YB_LAYER_THIN = 1, 2, 3, 4, 5


class YoloB200Error(RuntimeError):
    pass


if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} not found: build it with ./build.sh (or python -c 'import __graft_entry__ as g; g.build()'). "
        "yolov3_tensorflow_b200 has no CPU/PyTorch fallback.")

lib = C.CDLL(LIB_PATH)

vp, i32, f32, sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t


class ConvDesc(C.Structure):
    _fields_ = [(n, i32) for n in ("n", "h", "w", "cin", "cout", "ksize", "stride", "in_ld", "out_ld", "res_ld",
                                   "dtype", "out_fp32", "leaky", "upsample2x")]


class ConvSchedule(C.Structure):   # yb_conv_schedule_info
    _fields_ = [(n, i32) for n in ("pingpong", "consumers", "cluster", "block_m", "block_n", "block_k", "stages", "num_kb",
                                   "num_m_tiles", "num_n_tiles", "grid", "res_smem", "res_stages", "cluster_m",
                                   "cluster_n", "units", "epi_tma")]


class LayerSchedule(C.Structure):  # yb_layer_schedule_info
    _fields_ = [(n, i32) for n in ("igemm", "pingpong", "cluster_m", "cluster_n", "block_m", "block_n", "num_m_tiles",
                                   "num_n_tiles", "units", "max_clusters", "grid", "residual", "res_smem", "kernel",
                                   "epi_tma", "det_block_n")]


class WgradSchedule(C.Structure):  # yb_wgrad_schedule_info
    _fields_ = [(n, i32) for n in ("bnw", "tp", "stages", "num_kb", "kb_per_split", "splits", "tiles", "grid_x",
                                   "grid_y", "grid_z")]


class BnSchedule(C.Structure):     # yb_bn_schedule_info
    _fields_ = [(n, i32) for n in ("cpt", "r", "blocks_per_sm", "cv", "lanes")] + [("rows_per_block", C.c_long),
                                                                                    ("grid", i32)]


class LayerInfo(C.Structure):
    _fields_ = [(n, i32) for n in ("index", "cin", "cout", "ksize", "stride", "has_bn", "in_h", "in_w", "out_h",
                                   "out_w", "is_head", "scope_index", "upsample2x")]


class JpegInfo(C.Structure):       # yb_jpeg_info
    _fields_ = [(n, i32) for n in ("height", "width", "src_height", "src_width", "components", "h_samp", "v_samp",
                                   "restart_interval", "orientation", "mode")]


class JpegEncImage(C.Structure):   # yb_jpeg_enc_image
    _fields_ = [("pixels", vp), ("pitch", C.c_int64)] + [(n, i32) for n in (
        "height", "width", "channels", "quality", "luma_quality", "chroma_quality", "sampling", "restart_interval")]


class PlotLayout(C.Structure):     # yb_plot_layout
    _fields_ = [(n, i32) for n in ("length", "thickness", "text_w", "text_h", "rect_x1", "rect_y1", "org_x", "org_y")]


class AugmentParam(C.Structure):   # yb_augment_param
    _fields_ = [("out_offset", C.c_int64)] + [(n, i32) for n in (
        "out_h", "out_w", "crop_y", "crop_x", "canvas_h", "canvas_w", "off_y", "off_x", "src1", "src2")] + [
        ("w1", f32), ("w2", f32), ("color", i32), ("brightness", i32), ("hue", i32), ("saturation", f32),
        ("value", f32), ("fill", i32)]


class Optimizer(C.Structure):      # yb_optimizer
    _fields_ = [("kind", i32)] + [(n, f32) for n in ("lr", "grad_scale", "momentum", "decay", "beta1", "beta2", "epsilon",
                                                      "weight_decay", "clip_norm")]


_SIGS = {
    "yb_version": ([], i32),
    "yb_last_error_string": ([], C.c_char_p),
    "yb_set_option": ([C.c_char_p, C.c_char_p], i32),
    "yb_get_option": ([C.c_char_p], C.c_char_p),
    "yb_device_info": ([C.POINTER(i32)] * 3, i32),
    "yb_conv2d_fwd": ([C.POINTER(ConvDesc), vp, vp, vp, vp, vp, vp, vp, vp, vp], i32),
    "yb_conv2d_fwd_e4m3": ([C.POINTER(ConvDesc), vp, vp, vp, vp, vp, f32, vp, f32, vp], i32),
    "yb_conv_cout_pad": ([i32], i32),
    "yb_conv_schedule": ([C.POINTER(ConvDesc), i32, i32, i32, i32, C.POINTER(ConvSchedule)], i32),
    "yb_stem_conv_fwd": ([vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp, vp], i32),
    "yb_conv3x3_thin_fwd": ([C.POINTER(ConvDesc), vp, vp, vp, vp, vp, vp, vp], i32),
    "yb_conv3x3_halo_supported": ([C.POINTER(ConvDesc)], i32),
    "yb_conv3x3_halo_fwd": ([C.POINTER(ConvDesc), vp, vp, vp, vp, vp, vp, vp], i32),
    "yb_stem_conv1_fused_fwd": ([C.POINTER(ConvDesc), vp, vp, vp, vp, vp, vp, vp, vp, vp], i32),
    "yb_stem_conv_fwd_tc": ([vp, vp, vp, vp, i32, i32, i32, i32, i32, vp, vp], i32),
    "yb_stem_conv_fwd_tc_stats": ([vp, vp, vp, vp, i32, i32, i32, i32, i32, vp, vp, vp, vp], i32),
    "yb_process_box": ([vp, vp, vp, i32, i32, i32, i32, i32, C.POINTER(f32), vp, vp, vp, vp], i32),
    "yb_letterbox_params": ([i32, i32, i32, i32, C.POINTER(C.c_double), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)], i32),
    "yb_letterbox_normalize": ([vp, i32, i32, C.c_long, i32, i32, vp, vp], i32),
    "yb_resize_batch": ([vp, C.c_long, vp, vp, i32, i32, i32, i32, i32, vp, vp, vp], i32),
    "yb_resize_tables_bytes": ([vp, i32, i32, i32, i32, vp, C.POINTER(sz)], i32),
    "yb_resize_tables": ([vp, i32, i32, i32, i32, vp, vp, sz], i32),
    "yb_resize_batch_interp": ([vp, C.c_long, vp, vp, i32, i32, i32, i32, vp, vp, vp, sz, vp, vp, vp], i32),
    "yb_resize_boxes": ([vp, vp, i32, i32, i32, vp, i32, i32, i32, vp], i32),
    "yb_restore_boxes": ([vp, vp, i32, i32, i32, vp, vp], i32),
    "yb_augment_batch": ([vp, C.c_long, vp, vp, i32, vp, vp, i32, vp, C.c_long, vp, vp], i32),
    "yb_flip_batch": ([vp, i32, i32, i32, i32, vp, vp, vp, i32, i32, vp], i32),
    "yb_pack_conv_weights": ([vp, i32, i32, i32, i32, i32, i32, vp, vp], i32),
    "yb_pack_conv_weights_e4m3": ([vp, i32, i32, i32, i32, i32, vp, vp, vp], i32),
    "yb_amax": ([vp, C.c_long, C.c_long, i32, i32, vp, vp], i32),
    "yb_bn_fold": ([vp, vp, vp, vp, i32, f32, vp, vp, vp], i32),
    "yb_conv2d_wgrad": ([C.POINTER(ConvDesc), vp, vp, i32, i32, vp, vp], i32),
    "yb_stem_conv_wgrad": ([vp, vp, i32, i32, i32, i32, vp, vp], i32),
    "yb_stem_conv_wgrad_tc": ([vp, vp, i32, i32, i32, i32, vp, vp], i32),
    "yb_pack_dgrad_weights": ([vp, i32, i32, i32, i32, i32, i32, vp, vp], i32),
    "yb_pack_dgrad_weights_s2": ([vp, i32, i32, i32, i32, i32, vp, vp], i32),
    "yb_conv2d_dgrad_s2": ([vp, vp, i32, i32, vp, vp, i32, vp, i32, vp], i32),
    "yb_bn_finalize": ([vp, vp, C.c_long, i32, vp, vp, f32, f32, vp, vp, vp, vp, vp, vp, vp], i32),
    "yb_bn_act_apply": ([vp, C.c_long, vp, vp, vp, C.c_long, vp, C.c_long, i32, i32, i32, i32, i32, i32, i32, vp], i32),
    "yb_wgrad_schedule": ([C.POINTER(ConvDesc), i32, C.POINTER(WgradSchedule)], i32),
    "yb_bn_stats_act_apply": ([vp, C.c_long, vp, vp, vp, vp, f32, f32, vp, vp, vp, vp, vp, vp, vp, C.c_long, vp, C.c_long,
                               i32, i32, i32, i32, i32, i32, i32, vp], i32),
    "yb_bn_schedule": ([C.c_long, i32, i32, C.POINTER(BnSchedule)], i32),
    "yb_bn_bwd_reduce_workspace_bytes": ([C.POINTER(sz)], i32),
    "yb_bn_bwd_reduce": ([vp, C.c_long, vp, C.c_long, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, vp, vp, vp], i32),
    "yb_bn_bwd_apply": ([vp, C.c_long, vp, C.c_long, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, vp, C.c_long, vp], i32),
    "yb_col_sum": ([vp, C.c_long, C.c_long, i32, i32, vp, vp], i32),
    "yb_col_stats": ([vp, C.c_long, C.c_long, i32, i32, vp, vp, vp], i32),
    "yb_reorg_layer": ([vp, i32, i32, i32, i32, i32, i32, C.POINTER(f32), vp, vp, vp, vp, vp], i32),
    "yb_predict": ([vp, vp, vp, i32, i32, i32, i32, C.POINTER(f32), vp, vp, vp, vp, vp], i32),
    "yb_nms_workspace_bytes": ([i32, i32, i32, i32, C.POINTER(sz)], i32),
    "yb_nms": ([vp, vp, i32, i32, i32, i32, f32, f32, vp, sz, vp, vp, vp, vp, vp, vp], i32),
    "yb_voc_match": ([vp, vp, vp, vp, i32, i32, vp, vp, vp, i32, i32, C.c_double, vp, C.c_long, C.c_long, vp, vp], i32),
    "yb_voc_ap_workspace_bytes": ([C.c_long, i32, C.POINTER(sz)], i32),
    "yb_voc_ap": ([vp, C.c_long, vp, i32, i32, vp, sz, vp, vp], i32),
    "yb_kmeans_workspace_bytes": ([C.c_long, i32, C.POINTER(sz)], i32),
    "yb_kmeans_assign": ([vp, C.c_long, vp, i32, vp, vp, vp, vp, sz, vp], i32),
    "yb_kmeans_median": ([vp, C.c_long, vp, vp, i32, vp, vp, sz, vp], i32),
    "yb_kmeans_avg_iou": ([vp, C.c_long, vp, i32, vp, vp, sz, vp], i32),
    "yb_jpeg_parse": ([vp, sz, C.POINTER(JpegInfo)], i32),
    "yb_jpeg_pack_bytes": ([C.POINTER(vp), C.POINTER(sz), i32, C.POINTER(sz)], i32),
    "yb_jpeg_pack": ([C.POINTER(vp), C.POINTER(sz), i32, vp, sz, vp], i32),
    "yb_jpeg_workspace_bytes": ([vp, i32, C.POINTER(sz), C.POINTER(sz)], i32),
    "yb_jpeg_decode": ([vp, vp, i32, vp, vp, vp, vp, sz, vp], i32),
    "yb_jpeg_enc_header": ([C.POINTER(JpegEncImage), vp, sz, C.POINTER(sz)], i32),
    "yb_jpeg_enc_pack_bytes": ([C.POINTER(JpegEncImage), i32, C.POINTER(sz)], i32),
    "yb_jpeg_enc_pack": ([C.POINTER(JpegEncImage), i32, vp, sz], i32),
    "yb_jpeg_enc_workspace_bytes": ([vp, i32, C.POINTER(sz), C.POINTER(sz)], i32),
    "yb_jpeg_enc_encode": ([vp, vp, i32, vp, sz, vp, vp, sz, vp], i32),
    "yb_plot_label_layout": ([C.c_char_p, i32, i32, f32, i32, i32, i32, vp, C.POINTER(PlotLayout)], i32),
    "yb_plot_workspace_bytes": ([i32, i32, sz, C.POINTER(sz)], i32),
    "yb_plot_pack": ([vp, i32, vp, C.c_char_p, vp, i32, i32, vp, sz], i32),
    "yb_plot_boxes": ([vp, i32, i32, i32, vp, vp, vp, vp, i32, vp, vp, vp], i32),
    "yb_loss_workspace_bytes": ([i32, i32, i32, C.POINTER(sz)], i32),
    "yb_loss_layer": ([vp, vp, i32, i32, i32, i32, i32, i32, C.POINTER(f32), i32, i32, f32, f32, vp, sz, vp, vp, i32, i32, vp], i32),
    "yb_loss_finalize": ([vp, vp, vp], i32),
    "yb_box_iou": ([vp, vp, C.c_long, i32, vp, vp], i32),
    "yb_net_create": ([C.POINTER(vp), i32, i32, i32, i32, i32, i32], i32),
    "yb_net_destroy": ([vp], i32),
    "yb_net_num_layers": ([vp], i32),
    "yb_net_layer_info": ([vp, i32, C.POINTER(LayerInfo)], i32),
    "yb_net_layer_schedule": ([vp, i32, i32, C.POINTER(LayerSchedule)], i32),
    "yb_net_arena_bytes": ([vp, C.POINTER(sz), C.POINTER(sz)], i32),
    "yb_net_bind": ([vp, vp, sz, vp, sz, vp], i32),
    "yb_net_refold_bn": ([vp, vp], i32),
    "yb_net_set_conv_params": ([vp, i32, vp, i32, vp, vp, vp, vp, vp, vp], i32),
    "yb_net_forward": ([vp, vp, vp, vp, vp, vp], i32),
    "yb_net_detect_supported": ([vp], i32),
    "yb_net_detect_workspace_bytes": ([vp, i32, C.POINTER(sz)], i32),
    "yb_net_detect": ([vp, vp, C.POINTER(f32), i32, f32, f32, vp, sz, vp, vp, vp, vp, vp, vp, vp], i32),
    "yb_net_detect_phases": ([vp, vp, C.POINTER(f32), i32, f32, f32, vp, sz, vp, vp, vp, vp, vp, vp, i32, vp], i32),
    "yb_net_forward_layers": ([vp, vp, vp, vp, vp, i32, i32, vp], i32),
    "yb_net_train_fwd_bwd": ([vp, vp, vp, vp, vp, C.POINTER(f32), i32, i32, f32, f32, vp, vp, vp, vp, i32, vp], i32),
    "yb_net_train_backward": ([vp, vp, i32, i32, i32, vp], i32),
    "yb_net_grad_range": ([vp, i32, i32, C.POINTER(vp), C.POINTER(sz)], i32),
    "yb_net_train_forward_layer": ([vp, vp, i32, i32, i32, f32, vp, vp, vp, i32, vp], i32),
    "yb_net_train_loss": ([vp, vp, vp, vp, C.POINTER(f32), i32, i32, f32, vp, vp], i32),
    "yb_net_train_backward_layer": ([vp, vp, i32, i32, i32, i32, vp], i32),
    "yb_net_train_join": ([vp, vp], i32),
    "yb_net_bn_exchange_buffer": ([vp, i32, i32, C.POINTER(vp), C.POINTER(sz)], i32),
    "yb_net_bn_batch_stats": ([vp, i32] + [C.POINTER(vp)] * 4, i32),
    "yb_net_grad_buffer": ([vp, C.POINTER(vp), C.POINTER(sz)], i32),
    "yb_net_train_update": ([vp, C.POINTER(Optimizer), vp], i32),
    "yb_net_train_reset_state": ([vp, i32, vp], i32),
    "yb_net_opt_state": ([vp, C.POINTER(vp), C.POINTER(sz), C.POINTER(i32), C.POINTER(vp)], i32),
    "yb_net_opt_norms": ([vp, C.POINTER(vp), C.POINTER(i32)], i32),
    "yb_net_set_trainable": ([vp, i32, i32, vp], i32),
    "yb_net_train_refresh_dgrad": ([vp, vp], i32),
    "yb_net_get_conv_params": ([vp, i32] + [C.POINTER(vp)] * 6, i32),
    "yb_net_layer_grad": ([vp, i32] + [C.POINTER(vp)] * 4, i32),
    "yb_net_train_buffer": ([vp, i32, i32, C.POINTER(vp), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)], i32),
    "yb_net_layer_output": ([vp, i32, C.POINTER(vp), C.POINTER(i32), C.POINTER(i32)], i32),
    "yb_net_set_fp8_amax": ([vp, C.POINTER(f32), i32, vp], i32),
    "yb_net_fp8_layer_scales": ([vp, i32, C.POINTER(f32), C.POINTER(vp)], i32),
    "yb_net_forward_launches": ([vp], i32),
}
for _name, (_args, _ret) in _SIGS.items():
    _fn = getattr(lib, _name)          # AttributeError here == header/library mismatch: fail loudly
    _fn.argtypes = _args
    _fn.restype = _ret

EXPORTED = tuple(_SIGS)


def check(rc: int, what: str = ""):
    """Translate a yb_status into the Python exceptions the reference API raises."""
    if rc == 0:
        return
    msg = lib.yb_last_error_string().decode("utf-8", "replace")
    if rc == -1:
        raise ValueError(f"{what}: {msg}")
    raise YoloB200Error(f"{what}: status {rc}: {msg}")


def set_option(key: str, value):
    """Runtime switch of the library (include/yolob200.h: yb_set_option); value None restores the default."""
    check(lib.yb_set_option(key.encode(), None if value is None else str(value).encode()), f"yb_set_option({key})")


def get_option(key: str) -> str:
    return lib.yb_get_option(key.encode()).decode()


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_handle():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def fptr(values):
    arr = (f32 * len(values))(*[float(v) for v in values])
    return arr
