"""CPU tests: which layers of the 416^2 plans add a shortcut and which of them prefetch it into shared memory
(yb_net_layer_schedule on an unbound plan, yb_conv_schedule), and the YB_CONV_RES option.  No GPU needed."""
import ctypes as C

import pytest

KEYS = ("YB_CONV_RES", "YB_CONV_MCAST", "YB_CONV_PP", "YB_CONV_CTAS", "YB_CONV_EG", "YB_CONV_MODE", "YB_CONV_MC",
        "YB_CONV_EPI", "YB_HALO")
SMS = 132
# the 3x3 convs of the darknet residual blocks: Conv_3 (208^2, the halo kernel), Conv_6/8 (104^2), 8 at 52^2,
# 8 at 26^2, 4 at 13^2
RESIDUAL = [3, 6, 8] + list(range(11, 26, 2)) + list(range(28, 43, 2)) + list(range(45, 52, 2))


@pytest.fixture
def L():
    from yolov3_tensorflow_b200 import _lib
    for k in KEYS:
        _lib.set_option(k, None)
    yield _lib
    for k in KEYS:
        _lib.set_option(k, None)


def _plan_table(L, dtype, training=0, n=64, size=416):
    net = C.c_void_p()
    L.check(L.lib.yb_net_create(C.byref(net), 80, n, size, size, dtype, training), "net_create")
    try:
        rows = []
        for i in range(L.lib.yb_net_num_layers(net)):
            info, s = L.LayerInfo(), L.LayerSchedule()
            L.check(L.lib.yb_net_layer_info(net, i, C.byref(info)), "layer_info")
            L.check(L.lib.yb_net_layer_schedule(net, i, SMS, C.byref(s)), "layer_schedule")
            rows.append((info, s))
        return rows
    finally:
        L.lib.yb_net_destroy(net)


@pytest.mark.parametrize("dtype", ("f16", "bf16"))
def test_plan_residual_table(L, dtype):
    """Every shortcut layer of the 16-bit inference plan prefetches its shortcut: the halo kernel's Conv_3 with its
    halo tile, the others (all 3x3 ping-pong convs with 128-column tiles) during the main loop."""
    rows = _plan_table(L, L.YB_F16 if dtype == "f16" else L.YB_BF16)
    assert [info.index for info, s in rows if s.residual] == RESIDUAL
    for info, s in rows:
        i = info.index
        if i == 3:
            assert (s.igemm, s.residual, s.res_smem) == (0, 1, 1), "Conv_3 runs the halo kernel"
        elif s.residual:
            assert s.igemm and s.pingpong and s.block_n == 128 and info.ksize == 3 and info.stride == 1
            assert s.res_smem == 1, f"layer {i}"
        else:
            assert s.res_smem == 0, f"layer {i}"


def test_plan_residual_ldg_and_e4m3(L):
    """YB_CONV_RES=ldg: no prefetch anywhere, the same layers report their shortcut.  The e4m3 plan's igemm layers
    keep the global residual reads; its Conv_3 (fp16 in, e4m3 out, halo kernel) prefetches."""
    L.set_option("YB_CONV_RES", "ldg")
    rows = _plan_table(L, L.YB_F16)
    assert [info.index for info, s in rows if s.residual] == RESIDUAL
    assert not any(s.res_smem for _, s in rows)
    L.set_option("YB_CONV_RES", None)
    rows = _plan_table(L, L.YB_E4M3)
    assert [info.index for info, s in rows if s.residual] == RESIDUAL
    assert [info.index for info, s in rows if s.res_smem] == [3]


def test_training_plan_prefetches(L):
    """A training plan reports the prefetch at the same layers as the inference plans."""
    rows = _plan_table(L, L.YB_BF16, training=1, n=32)
    assert [info.index for info, s in rows if s.res_smem] == RESIDUAL


def _conv_schedule(L, **kw):
    d = dict(n=8, h=52, w=52, cin=128, cout=256, ksize=3, stride=1, in_ld=128, out_ld=256, res_ld=256,
             dtype=L.YB_F16, out_fp32=0, leaky=1, upsample2x=0)
    d.update(kw)
    desc = L.ConvDesc(**d)
    info = L.ConvSchedule()
    rc = L.lib.yb_conv_schedule(C.byref(desc), 0, 0, 0, SMS, C.byref(info))
    return rc, info


def test_conv_schedule_reports_the_path(L):
    rc, i = _conv_schedule(L)
    assert rc == 0 and i.pingpong and i.res_smem == 1
    assert (i.stages, i.res_stages) == (6, 4)          # 2 x 32 KB shortcut tiles take two 32 KB ring stages
    rc, i = _conv_schedule(L, dtype=L.YB_BF16, n=3, h=20, w=20)
    assert rc == 0 and i.res_smem == 1
    # not where the epilogue keeps its global read: 64-column tiles, 32-channel k-blocks, the cooperative schedule,
    # a 2x-upsampled output
    for kw in (dict(cout=64, out_ld=64, res_ld=64), dict(cin=96, in_ld=96), dict(ksize=1, cin=256, in_ld=256),
               dict(upsample2x=1)):
        rc, i = _conv_schedule(L, **kw)
        assert rc == 0 and i.res_smem == 0 and i.res_stages == i.stages, kw
    L.set_option("YB_CONV_PP", "0")
    rc, i = _conv_schedule(L)
    assert rc == 0 and i.pingpong == 0 and i.res_smem == 0
    L.set_option("YB_CONV_PP", None)
    L.set_option("YB_CONV_RES", "ldg")
    rc, i = _conv_schedule(L)
    assert rc == 0 and i.res_smem == 0
    L.set_option("YB_CONV_RES", "smem")
    rc, i = _conv_schedule(L)
    assert rc == 0 and i.res_smem == 1
    for bad in ("tma", "LDG", "1"):
        L.set_option("YB_CONV_RES", bad)
        assert _conv_schedule(L)[0] != 0
