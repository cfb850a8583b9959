"""The shortcut prefetch of the implicit-GEMM conv (csrc/conv_igemm.cu, YB_CONV_RES) on the GPU.

With YB_CONV_RES=smem the ping-pong kernel TMA-loads each work unit's residual tile into its warpgroup's shared-memory
tile during the unit's main loop, and the epilogue adds it from there; with ldg the epilogue reads it from global
memory.  Both add the same values in the same order, so every output must be byte-identical between the two, and
within the float64 bound of tests/conv_ref.py.  Cases: every shortcut shape of the 416^2 plan at batch 8 in fp16 and
bf16, without and with multicast clusters; the 52^2 shape at batch 64; a partial last m-tile; an in-place residual
whose row pitch exceeds cout; grids capped to a few CTAs, so that each warpgroup refills its shortcut tile dozens of
times; and the whole batch-64 detect step of the plan.  The halo kernel (Conv_3: 32 -> 64, 3x3, stride 1) loads its
residual box with each tile's halo instead: fp16, bf16, partial bottom tiles, an in-place residual, and the fp8 plan,
whose Conv_3 runs the e4m3-output instantiation."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from tests import conv_ref as R
from tests.test_gpu_conv_schedule import GUARD, FwdCase, _guards

pytestmark = pytest.mark.gpu

KEYS = ("YB_CONV_RES", "YB_CONV_MCAST", "YB_CONV_PP", "YB_CONV_CTAS", "YB_CONV_EG", "YB_CONV_MODE", "YB_CONV_MC",
        "YB_CONV_EPI")


@pytest.fixture
def L():
    from yolov3_tensorflow_b200 import _lib
    for k in KEYS:
        _lib.set_option(k, None)
    yield _lib
    for k in KEYS:
        _lib.set_option(k, None)


def _schedule(L, d):
    s = C.c_int()
    L.check(L.lib.yb_device_info(C.byref(s), None, None), "device_info")
    info = L.ConvSchedule()
    L.check(L.lib.yb_conv_schedule(C.byref(d), 0, 0, 0, s.value, C.byref(info)), "conv_schedule")
    return info


def _res_ab(L, name, case, mcast=None, cap=None, min_upw=0):
    """The case with YB_CONV_RES=ldg (checked against float64), then with smem: byte-identical outputs."""
    L.set_option("YB_CONV_MCAST", mcast)
    L.set_option("YB_CONV_CTAS", cap)
    outs = {}
    for mode in ("ldg", "smem"):
        L.set_option("YB_CONV_RES", mode)
        i = _schedule(L, case.desc)
        assert i.pingpong == 1 and i.res_smem == (mode == "smem"), f"{name} {mode}: schedule"
        upw = R.units_per_warpgroup(i)
        assert upw >= min_upw, f"{name}: only {upw} units per warpgroup"
        buf, ssum, ssq = case.run()
        if mode == "ldg":
            outs[mode], worst = case.check(f"{name} ldg", buf, ssum, ssq, upw, i.grid)
        else:
            _guards(f"{name} smem", buf, case.rows, case.out_off, case.cout)
            outs[mode] = buf[GUARD:GUARD + case.rows, case.out_off:case.out_off + case.cout].clone()
            print(f"RES {name} mcast={mcast} cap={cap}: cluster {i.cluster} grid {i.grid} units/wg {upw} "
                  f"stages {i.res_stages} worst {worst:.3f}")
    assert torch.equal(outs["ldg"].view(torch.int16), outs["smem"].view(torch.int16)), \
        f"{name} mcast={mcast} cap={cap}: the shared-memory shortcut changed the output bits"


DT = (torch.float16, torch.bfloat16)
_dt_id = {torch.float16: "f16", torch.bfloat16: "bf16"}

# (n, h, w, cin, cout): the shortcut convs of the 416^2 plan (3x3, stride 1) at batch 8
SHORTCUT_SHAPES = {
    "104_64_128": (8, 104, 104, 64, 128),
    "52_128_256": (8, 52, 52, 128, 256),
    "26_256_512": (8, 26, 26, 256, 512),
    "13_512_1024": (8, 13, 13, 512, 1024),
}


@pytest.mark.parametrize("dtype", DT, ids=_dt_id.get)
@pytest.mark.parametrize("name", list(SHORTCUT_SHAPES))
def test_res_plan_shapes_bit_identical(L, name, dtype):
    n, h, w, cin, cout = SHORTCUT_SHAPES[name]
    case = FwdCase(L, n, h, w, cin, cout, 3, 1, dtype=dtype, res="sep", seed=list(SHORTCUT_SHAPES).index(name) + 40)
    for mcast in ("0", "2x1", "2x2"):
        _res_ab(L, name, case, mcast=mcast)


@pytest.mark.parametrize("dtype", DT, ids=_dt_id.get)
def test_res_52_batch64_bit_identical(L, dtype):
    case = FwdCase(L, 64, 52, 52, 128, 256, 3, 1, dtype=dtype, res="sep", seed=50)
    for mcast in ("0", "2x2"):
        _res_ab(L, "52_128_256_b64", case, mcast=mcast)


@pytest.mark.parametrize("dtype", DT, ids=_dt_id.get)
def test_res_partial_tile_and_capped_grid(L, dtype):
    """3 x 20 x 20 = 1200 pixels = 9.4 m-tiles: the last tile is partial, and under 2 x 1 / 2 x 2 clusters the last
    cluster has an idle rank.  cin 192: 27 k-blocks, not a multiple of the 4-stage ring.  Capped grids: every
    warpgroup takes several units, one CTA takes all of them."""
    case = FwdCase(L, 3, 20, 20, 192, 256, 3, 1, dtype=dtype, res="sep", seed=51)
    for mcast in ("0", "2x1", "2x2"):
        _res_ab(L, "partial", case, mcast=mcast)
    for mcast, cap in (("0", "1"), ("0", "3"), ("2x1", "2"), ("2x2", "4")):
        _res_ab(L, "partial", case, mcast=mcast, cap=cap, min_upw=2)


@pytest.mark.parametrize("dtype", DT, ids=_dt_id.get)
def test_res_buffer_reuse_many_units(L, dtype):
    """104^2 x 2 images, 169 m-tiles, on one CTA / one cluster: each warpgroup reuses its shortcut tile 20-85 times."""
    case = FwdCase(L, 2, 104, 104, 64, 128, 3, 1, dtype=dtype, res="sep", seed=52)
    for mcast, cap in (("0", "1"), ("0", "2"), ("2x1", "2"), ("2x2", "4")):
        _res_ab(L, "reuse", case, mcast=mcast, cap=cap, min_upw=20)


def test_res_inplace_wide_pitch(L):
    """The residual is the output itself (in place), in a buffer of row pitch cout + 64."""
    case = FwdCase(L, 2, 26, 26, 128, 256, 3, 1, dtype=torch.float16, res="inplace", out_extra=64, seed=53)
    assert case.desc.res_ld > case.desc.cout
    for mcast, cap in (("0", None), ("2x2", None), ("0", "2")):
        _res_ab(L, "inplace", case, mcast=mcast, cap=cap)


def test_res_stats_bit_identical(L):
    """BN statistics on (the training forward's m-fastest unit order): same output bits, sums within the bound."""
    case = FwdCase(L, 2, 26, 26, 128, 256, 3, 1, res="sep", stats=True, seed=54)
    _res_ab(L, "stats", case)
    _res_ab(L, "stats", case, cap="3")


def _layer_schedules(L, plan):
    out = []
    for i in range(plan.num_layers):
        s = L.LayerSchedule()
        L.check(L.lib.yb_net_layer_schedule(plan.handle, i, 0, C.byref(s)), "layer_schedule")
        out.append(s)
    return out


def test_res_detect_step_bit_identical(L):
    """yb_net_forward and yb_net_detect at batch 64, 416^2 with bench weights: YB_CONV_RES=ldg against the default
    (smem), byte for byte.  The option is captured when the plan binds."""
    import yolov3_tensorflow_b200 as pkg
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    from bench import make_bench_params
    anchors = pkg.parse_anchors(os.path.join(root, "yolov3_tensorflow_b200", "data", "yolo_anchors.txt"))
    params = make_bench_params(specs=pkg.yolov3.conv_table(80))
    x = torch.from_numpy(np.random.default_rng(4).random((64, 416, 416, 3), dtype=np.float32)).cuda()
    outs, prefetched = {}, {}
    for mode in ("ldg", None):
        L.set_option("YB_CONV_RES", mode)
        m = pkg.yolov3(80, anchors, dtype="fp16")
        m.set_params(params, "HWIO")
        fms = [t.cpu().clone() for t in m.forward(x)]
        boxes, ob, os_, ol, oi, cnt = (t.cpu().clone() for t in m.detect_raw(x, max_boxes=200, score_thresh=0.3,
                                                                            nms_thresh=0.45))
        valid = torch.arange(ob.shape[1])[None, :] < cnt[:, None].long()
        outs[mode] = fms + [boxes, cnt, ob[valid], os_[valid], ol[valid], oi[valid]]
        prefetched[mode] = sum(s.res_smem for s in _layer_schedules(L, m._last_plan))
        del m
    assert prefetched["ldg"] == 0 and prefetched[None] == 23, prefetched      # 22 igemm layers + the halo Conv_3
    assert int(outs["ldg"][4].sum()) > 0, "no detections: the comparison would be empty"
    for k, (a, b) in enumerate(zip(outs["ldg"], outs[None])):
        assert a.dtype == b.dtype and a.shape == b.shape, f"output {k}"
        assert torch.equal(a.view(torch.uint8) if a.is_floating_point() else a,
                           b.view(torch.uint8) if b.is_floating_point() else b), f"output {k} differs"


def _halo_run(L, case):
    buf = torch.full((GUARD + case.rows + GUARD, case.out_ld), -7.0, dtype=case.odt, device="cuda")
    op = buf.data_ptr() + (GUARD * case.out_ld + case.out_off) * 2
    if case.res_mode == "inplace":
        buf[GUARD:GUARD + case.rows, case.out_off:case.out_off + case.cout] = case.prev
        resp = C.c_void_p(op)
    else:
        resp = L.ptr(case.prev)
    assert L.lib.yb_conv3x3_halo_supported(C.byref(case.desc)) == 1
    L.check(L.lib.yb_conv3x3_halo_fwd(C.byref(case.desc), C.c_void_p(case.xp), L.ptr(case.wp), L.ptr(case.sc),
                                      L.ptr(case.sh), resp, C.c_void_p(op), L.stream_handle()), "conv_halo")
    torch.cuda.synchronize()
    return buf


# (n, h, w, extras): Conv_3's shape (208^2 at batch 2), a partial bottom tile row (20 % 16), an in-place residual of
# row pitch cout + 64
HALO_CASES = {
    "208": (2, 208, 208, {}),
    "partial": (3, 20, 24, {}),
    "inplace": (2, 40, 32, dict(res="inplace", out_extra=64)),
}


@pytest.mark.parametrize("dtype", DT, ids=_dt_id.get)
@pytest.mark.parametrize("name", list(HALO_CASES))
def test_res_halo_bit_identical(L, name, dtype):
    n, h, w, kw = HALO_CASES[name]
    kw = dict(res="sep", **kw) if "res" not in kw else kw
    case = FwdCase(L, n, h, w, 32, 64, 3, 1, dtype=dtype, seed=60 + list(HALO_CASES).index(name), **kw)
    outs = {}
    for mode in ("ldg", "smem"):
        L.set_option("YB_CONV_RES", mode)
        buf = _halo_run(L, case)
        if mode == "ldg":
            outs[mode], worst = case.check(f"halo {name} ldg", buf, None, None, 0, 1)
        else:
            _guards(f"halo {name} smem", buf, case.rows, case.out_off, case.cout)
            outs[mode] = buf[GUARD:GUARD + case.rows, case.out_off:case.out_off + case.cout].clone()
    print(f"RES halo {name}: worst {worst:.3f}")
    assert torch.equal(outs["ldg"].view(torch.int16), outs["smem"].view(torch.int16)), \
        f"halo {name}: the prefetched residual changed the output bits"


def test_res_fp8_plan_bit_identical(L):
    """The fp8 plan (its Conv_3 is the halo kernel's e4m3-output instantiation, fp16 residual): every feature map and
    the detections of YB_CONV_RES=ldg and smem, byte for byte."""
    import yolov3_tensorflow_b200 as pkg
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    from bench import make_bench_params
    anchors = pkg.parse_anchors(os.path.join(root, "yolov3_tensorflow_b200", "data", "yolo_anchors.txt"))
    params = make_bench_params(specs=pkg.yolov3.conv_table(80))
    x = torch.from_numpy(np.random.default_rng(5).random((4, 416, 416, 3), dtype=np.float32)).cuda()
    outs, conv3 = {}, {}
    for mode in ("ldg", "smem"):
        L.set_option("YB_CONV_RES", mode)
        m = pkg.yolov3(80, anchors, dtype="fp16")
        m.set_params(params, "HWIO")
        qm = m.quantize_fp8([x])
        fms = [t.cpu().clone() for t in qm.forward(x)]
        boxes, ob, os_, ol, oi, cnt = (t.cpu().clone() for t in qm.detect_raw(x, max_boxes=200, score_thresh=0.3,
                                                                             nms_thresh=0.45))
        valid = torch.arange(ob.shape[1])[None, :] < cnt[:, None].long()
        outs[mode] = fms + [boxes, cnt, ob[valid], os_[valid], ol[valid], oi[valid]]
        conv3[mode] = _layer_schedules(L, qm._last_plan)[3]
        del m, qm
    assert (conv3["ldg"].igemm, conv3["ldg"].residual, conv3["ldg"].res_smem) == (0, 1, 0)
    assert (conv3["smem"].igemm, conv3["smem"].residual, conv3["smem"].res_smem) == (0, 1, 1)
    for k, (a, b) in enumerate(zip(outs["ldg"], outs["smem"])):
        assert a.dtype == b.dtype and a.shape == b.shape, f"output {k}"
        assert torch.equal(a.view(torch.uint8) if a.is_floating_point() else a,
                           b.view(torch.uint8) if b.is_floating_point() else b), f"fp8 plan output {k} differs"
