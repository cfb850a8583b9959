"""Ping-pong multicast clusters of the implicit-GEMM conv (csrc/conv_igemm.cu, YB_CONV_MCAST) on the GPU.

A CM x CN cluster only changes where each CTA's operand bytes come from: every CTA still receives its whole A and B
tiles and runs the same wgmma sequence over them.  So every clustered output must be byte-identical to the unclustered
one on the same operands, and within the float64 bound of tests/conv_ref.py.  Sentinel rows around the output and the
columns outside a written channel slice must keep their sentinel.  Cases: every 3x3 and 1x1 conv shape of the 416^2
inference plan at batch 8, the 52^2 3x3 layers at batch 64, residual, concat slice, 2x upsample, stride 2, an odd
number of m-tiles (the last cluster half idle) and a grid capped to one cluster (every warpgroup wraps the ring many
times).  The cooperative schedule's clusters (YB_CONV_MODE=2cta, 2 x 1 or 4 x 1) share the same loads and release, so
the plan shapes and the tails run them too, against the unclustered cooperative bits.  Then the whole batch-64 detect
step of the plan, multicast on against off."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import conv_ref as R
from tests.test_gpu_conv_schedule import GUARD, FwdCase, _guards

pytestmark = pytest.mark.gpu

KEYS = ("YB_CONV_MCAST", "YB_CONV_PP", "YB_CONV_CTAS", "YB_CONV_EG", "YB_CONV_MODE", "YB_CONV_MC", "YB_CONV_EPI")
SHAPES = ("2x1", "1x2", "2x2")


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


def _out(case, buf):
    _guards("mcast", buf, case.rows, case.out_off, case.cout)
    return buf[GUARD:GUARD + case.rows, case.out_off:case.out_off + case.cout].clone()


def _mcast_sweep(L, name, case, pp=None, cap=None, want_cluster=None):
    """The case unclustered, then under every forced shape: byte-identical outputs, float64 bound on the first."""
    L.set_option("YB_CONV_PP", pp)
    L.set_option("YB_CONV_CTAS", cap)
    L.set_option("YB_CONV_MCAST", "0")
    i0 = _schedule(L, case.desc)
    assert i0.cluster == 1
    buf, ssum, ssq = case.run()
    base, worst = case.check(f"{name} mcast=0", buf, ssum, ssq, R.units_per_warpgroup(i0), i0.grid)
    tiles_n = i0.num_n_tiles
    for shape in SHAPES:
        L.set_option("YB_CONV_MCAST", shape)
        i = _schedule(L, case.desc)
        cm, cn = int(shape[0]), int(shape[2])
        if tiles_n % 2:
            cn = 1
        if i.pingpong:
            assert i.cluster == cm * cn, f"{name} {shape}: cluster {i.cluster}"
            assert i.grid % i.cluster == 0
        if want_cluster is not None:
            assert i.cluster == want_cluster[shape], f"{name} {shape}: cluster {i.cluster}"
        buf, _, _ = case.run()
        got = _out(case, buf)
        assert torch.equal(got, base), f"{name} {shape}: output differs from the unclustered bits"
        print(f"MCAST {name} {shape}: {'pp' if i.pingpong else 'coop'} cluster {i.cluster} grid {i.grid} "
              f"tiles {i.num_m_tiles}x{i.num_n_tiles} num_kb {i.num_kb} worst {worst:.3f}")


def _coop_sweep(L, name, case, cap=None):
    """The cooperative schedule unclustered, then in its 2 x 1 and 4 x 1 clusters (YB_CONV_MODE=2cta, YB_CONV_MC=1),
    which load and release the ring like the ping-pong clusters: byte-identical outputs, float64 bound on the first."""
    L.set_option("YB_CONV_PP", "0")
    L.set_option("YB_CONV_CTAS", cap)
    i0 = _schedule(L, case.desc)
    assert i0.cluster == 1 and not i0.pingpong
    buf, ssum, ssq = case.run()
    base, worst = case.check(f"{name} coop", buf, ssum, ssq, R.units_per_warpgroup(i0), i0.grid)
    for mc, cs in ((None, 2), ("1", 4)):
        L.set_option("YB_CONV_MODE", "2cta")
        L.set_option("YB_CONV_MC", mc)
        i = _schedule(L, case.desc)
        assert i.cluster == cs and not i.pingpong and i.grid % cs == 0, f"{name} coop {cs}: cluster {i.cluster}"
        buf, _, _ = case.run()
        assert torch.equal(_out(case, buf), base), f"{name} coop {cs}: output differs from the unclustered bits"
        print(f"COOP {name} {cs}x1: grid {i.grid} tiles {i.num_m_tiles}x{i.num_n_tiles} num_kb {i.num_kb} "
              f"worst {worst:.3f}")
    L.set_option("YB_CONV_MODE", None)
    L.set_option("YB_CONV_MC", None)


DT = (torch.float16, torch.bfloat16)
_dt_id = {torch.float16: "f16", torch.bfloat16: "bf16"}

# (n, h, w, cin, cout, k, s, extras): the conv shapes of the 416^2 plan (conv_igemm layers) at batch 8
PLAN_SHAPES = {
    "3x3s2_208_64_128": (8, 208, 208, 64, 128, 3, 2, {}),
    "3x3_104_64_128_res": (8, 104, 104, 64, 128, 3, 1, dict(res="sep")),
    "3x3s2_104_128_256": (8, 104, 104, 128, 256, 3, 2, {}),
    "3x3_52_128_256_res": (8, 52, 52, 128, 256, 3, 1, dict(res="sep")),
    "3x3s2_52_256_512": (8, 52, 52, 256, 512, 3, 2, {}),
    "3x3_26_256_512_res": (8, 26, 26, 256, 512, 3, 1, dict(res="sep")),
    "3x3s2_26_512_1024": (8, 26, 26, 512, 1024, 3, 2, {}),
    "3x3_13_512_1024_res": (8, 13, 13, 512, 1024, 3, 1, dict(res="sep")),
    "3x3_52_128_256_slice": (8, 52, 52, 128, 256, 3, 1, dict(out_extra=128)),     # the route1 store into cat2
    "1x1_208_64_32": (8, 208, 208, 64, 32, 1, 1, {}),
    "1x1_104_128_64": (8, 104, 104, 128, 64, 1, 1, {}),
    "1x1_52_256_128": (8, 52, 52, 256, 128, 1, 1, {}),
    "1x1_26_768_256": (8, 26, 26, 768, 256, 1, 1, {}),
    "1x1_13_1024_512": (8, 13, 13, 1024, 512, 1, 1, {}),
    "1x1_13_512_256_up_slice": (8, 13, 13, 512, 256, 1, 1, dict(upsample=True, out_extra=512)),
    "1x1_26_256_128_up_slice": (8, 26, 26, 256, 128, 1, 1, dict(upsample=True, out_extra=256)),
    "1x1_52_256_255_head": (8, 52, 52, 256, 255, 1, 1, dict(out_fp32=True, leaky=False)),
}


@pytest.mark.parametrize("dtype", DT, ids=_dt_id.get)
@pytest.mark.parametrize("name", list(PLAN_SHAPES))
def test_mcast_plan_shapes_bit_identical(L, name, dtype):
    n, h, w, cin, cout, k, s, kw = PLAN_SHAPES[name]
    case = FwdCase(L, n, h, w, cin, cout, k, s, dtype=dtype, seed=list(PLAN_SHAPES).index(name), **kw)
    # ping-pong as the plan runs it; the 1x1 convs with 128-column tiles (cooperative by default) also forced to
    # ping-pong, so that the clustered 2D-tile loads of A run too
    _mcast_sweep(L, name, case)
    if k == 1 and not case.desc.out_fp32 and L.lib.yb_conv_cout_pad(cout) % 128 == 0:
        _mcast_sweep(L, name + " pp=1", case, pp="1")
    _coop_sweep(L, name, case)


@pytest.mark.parametrize("dtype", DT, ids=_dt_id.get)
def test_mcast_52_batch64_bit_identical(L, dtype):
    for name, kw in (("3x3_52_128_256_res_b64", dict(res="sep")), ("3x3s2_104_128_256_b64", {})):
        if "s2" in name:
            case = FwdCase(L, 64, 104, 104, 128, 256, 3, 2, dtype=dtype, seed=11, **kw)
        else:
            case = FwdCase(L, 64, 52, 52, 128, 256, 3, 1, dtype=dtype, seed=12, **kw)
        _mcast_sweep(L, name, case)


@pytest.mark.parametrize("dtype", DT, ids=_dt_id.get)
@pytest.mark.parametrize("cin", (128, 192))
def test_mcast_tails_and_capped_grid(L, cin, dtype):
    """24 x 24 pixels = 4.5 m-tiles (5: the last 2-row cluster has one idle m-tile), two n-tiles; cin 192 gives
    27 k-blocks (not a multiple of the ring depth).  Capped to one cluster, every warpgroup runs >= 3 units."""
    case = FwdCase(L, 1, 24, 24, cin, 256, 3, 1, dtype=dtype, res="sep", seed=cin)
    _mcast_sweep(L, f"tail cin{cin}", case)
    for cap in ("4", "2"):
        _mcast_sweep(L, f"tail cin{cin} cap{cap}", case, cap=cap)
    _coop_sweep(L, f"tail cin{cin}", case)
    _coop_sweep(L, f"tail cin{cin} cap4", case, cap="4")
    # stride 2, batch tail inside a tile
    case = FwdCase(L, 3, 20, 20, cin, 256, 3, 2, dtype=dtype, seed=cin + 1)
    _mcast_sweep(L, f"tail s2 cin{cin}", case, cap="4")


def test_mcast_stats_bit_identical(L):
    """BN statistics (m-fastest unit order) under the forced shapes: same conv output bits, sums within the bound."""
    case = FwdCase(L, 2, 26, 26, 128, 256, 3, 1, stats=True, seed=5)
    _mcast_sweep(L, "stats", case)


def test_mcast_option_rejects_bad_value(L):
    case_desc = L.ConvDesc(n=1, h=26, w=26, cin=128, cout=256, ksize=3, stride=1, in_ld=128, out_ld=256, res_ld=0,
                           dtype=L.YB_F16, out_fp32=0, leaky=1, upsample2x=0)
    L.set_option("YB_CONV_MCAST", "3x3")
    info = L.ConvSchedule()
    assert L.lib.yb_conv_schedule(C.byref(case_desc), 0, 0, 0, 132, C.byref(info)) != 0


def _plan_schedule(L, plan, sm_count=0):
    out = []
    for i in range(plan.num_layers):
        s = L.LayerSchedule()
        L.check(L.lib.yb_net_layer_schedule(plan.handle, i, sm_count, C.byref(s)), "layer_schedule")
        out.append(s)
    return out


def test_mcast_detect_step_bit_identical(L):
    """yb_net_detect at batch 64, 416^2 with bench weights: the plan rule against YB_CONV_MCAST=0, byte for byte.  The
    plan's schedule on this device: grids whole clusters, no more than cudaOccupancyMaxActiveClusters of them."""
    import os
    import sys
    import yolov3_tensorflow_b200 as pkg
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    from bench import make_bench_params
    anchors = pkg.parse_anchors(os.path.join(root, "yolov3_tensorflow_b200", "data", "yolo_anchors.txt"))
    params = make_bench_params(specs=pkg.yolov3.conv_table(80))
    x = torch.from_numpy(np.random.default_rng(3).random((64, 416, 416, 3), dtype=np.float32)).cuda()
    outs, scheds = {}, {}
    for mc in ("0", None):
        L.set_option("YB_CONV_MCAST", mc)
        m = pkg.yolov3(80, anchors, dtype="fp16")
        m.set_params(params, "HWIO")
        fms = [t.cpu().clone() for t in m.forward(x)]           # every layer's output feeds these (heads unfused)
        boxes, ob, os_, ol, oi, cnt = (t.cpu().clone() for t in m.detect_raw(x, max_boxes=200, score_thresh=0.3,
                                                                            nms_thresh=0.45))
        valid = torch.arange(ob.shape[1])[None, :] < cnt[:, None].long()   # slots past a count hold no result
        outs[mc] = fms + [boxes, cnt, ob[valid], os_[valid], ol[valid], oi[valid]]
        scheds[mc] = _plan_schedule(L, m._last_plan)
        del m
    assert int(outs["0"][4].sum()) > 0, "no detections: the comparison would be empty"
    for k, (a, b) in enumerate(zip(outs["0"], outs[None])):
        assert a.dtype == b.dtype and a.shape == b.shape, f"output {k}"
        assert torch.equal(a.view(torch.uint8) if a.is_floating_point() else a,
                           b.view(torch.uint8) if b.is_floating_point() else b), f"output {k} differs with multicast on"
    clustered = 0
    for i, s in enumerate(scheds[None]):
        if not s.igemm:
            continue
        cs = s.cluster_m * s.cluster_n
        assert s.grid % cs == 0 and s.grid <= s.max_clusters * cs, f"layer {i}: grid {s.grid}, cluster {cs}"
        assert scheds["0"][i].cluster_m * scheds["0"][i].cluster_n == 1
        clustered += cs > 1
        print(f"PLAN layer {i}: {s.cluster_m}x{s.cluster_n} pp {s.pingpong} units {s.units} grid {s.grid} "
              f"max clusters {s.max_clusters}")
    assert clustered > 0
