"""CPU tests: the multicast-cluster shapes the 416^2 plans choose per layer (yb_net_layer_schedule on an unbound plan),
and the YB_CONV_MCAST option.  No GPU needed: an unbound plan and a given SM count use the host model of the grid."""
import ctypes as C

import pytest

KEYS = ("YB_CONV_MCAST", "YB_CONV_PP", "YB_CONV_CTAS", "YB_CONV_EG", "YB_CONV_MODE", "YB_CONV_MC", "YB_CONV_EPI",
        "YB_HALO")
SMS = 132


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


def _check_grid(i, s):
    cs = s.cluster_m * s.cluster_n
    assert s.max_clusters == SMS // cs
    assert s.grid % cs == 0 and 0 < s.grid <= s.max_clusters * cs, f"layer {i}: grid {s.grid}, cluster {cs}"
    assert s.units == -(-s.num_m_tiles // s.cluster_m) * (s.num_n_tiles // s.cluster_n)
    assert s.grid == min(s.units, s.max_clusters) * cs


@pytest.mark.parametrize("dtype", ("f16", "bf16"))
def test_plan_rule_per_layer(L, dtype):
    code = L.YB_F16 if dtype == "f16" else L.YB_BF16
    rows = _plan_table(L, code)
    assert len(rows) == 75
    shapes = {}
    for info, s in rows:
        i = info.index
        if i == 0 or (info.ksize == 3 and info.cin == 32):
            assert s.igemm == 0, f"layer {i}: the stem and the Cin = 32 layers run the halo kernel"
            continue
        assert s.igemm == 1
        _check_grid(i, s)
        if info.ksize == 3:
            assert s.pingpong == 1
            want = (2, 2) if s.num_n_tiles % 2 == 0 else (2, 1)
        else:
            want = (1, 1)
        assert (s.cluster_m, s.cluster_n) == want, f"layer {i} ({info.cin}->{info.cout} k{info.ksize} " \
                                                   f"@{info.out_h}): {s.cluster_m}x{s.cluster_n}"
        shapes.setdefault((info.ksize, info.out_h), set()).add((s.cluster_m, s.cluster_n))
    # the 3x3 layers by output size: 104^2 one n-tile (2 x 1), 52^2 / 26^2 / 13^2 2 / 4 / 8 n-tiles (2 x 2)
    assert shapes[(3, 104)] == {(2, 1)}
    assert shapes[(3, 52)] == shapes[(3, 26)] == shapes[(3, 13)] == {(2, 2)}


def test_plan_rule_off(L):
    """YB_CONV_MCAST=0, training plans and the e4m3 plan: no multicast cluster anywhere."""
    L.set_option("YB_CONV_MCAST", "0")
    plans = [_plan_table(L, L.YB_F16)]
    L.set_option("YB_CONV_MCAST", None)
    plans += [_plan_table(L, L.YB_BF16, training=1, n=32), _plan_table(L, L.YB_E4M3)]
    for rows in plans:
        for info, s in rows:
            if s.igemm:
                assert (s.cluster_m, s.cluster_n) == (1, 1), f"layer {info.index}"
                _check_grid(info.index, s)


@pytest.mark.parametrize("shape", ("2x1", "1x2", "2x2"))
def test_forced_shape(L, shape):
    """A forced shape applies to every 16-bit ping-pong launch, the single convs of yb_conv2d_fwd included; CN = 2
    only where the n-tile count is even; the cooperative launches keep no cluster."""
    L.set_option("YB_CONV_MCAST", shape)
    cm, cn = int(shape[0]), int(shape[2])
    for info, s in _plan_table(L, L.YB_F16):
        if not s.igemm:
            continue
        _check_grid(info.index, s)
        if s.pingpong:
            assert (s.cluster_m, s.cluster_n) == (cm, cn if s.num_n_tiles % 2 == 0 else 1), f"layer {info.index}"
        else:
            assert (s.cluster_m, s.cluster_n) == (1, 1)
    d = L.ConvDesc(n=8, h=52, w=52, cin=128, cout=256, ksize=3, stride=1, in_ld=128, out_ld=256, res_ld=0,
                   dtype=L.YB_F16, out_fp32=0, leaky=1, upsample2x=0)
    info = L.ConvSchedule()
    L.check(L.lib.yb_conv_schedule(C.byref(d), 0, 0, 0, SMS, C.byref(info)), "conv_schedule")
    assert info.pingpong == 1 and info.cluster == cm * cn and info.grid % info.cluster == 0
    assert (info.cluster_m, info.cluster_n) == (cm, cn)
    assert info.units == -(-info.num_m_tiles // cm) * (info.num_n_tiles // cn)
    assert info.grid == min(info.units, SMS // info.cluster) * info.cluster


def test_single_conv_default_unclustered(L):
    d = L.ConvDesc(n=8, h=52, w=52, cin=128, cout=256, ksize=3, stride=1, in_ld=128, out_ld=256, res_ld=0,
                   dtype=L.YB_F16, out_fp32=0, leaky=1, upsample2x=0)
    info = L.ConvSchedule()
    L.check(L.lib.yb_conv_schedule(C.byref(d), 0, 0, 0, SMS, C.byref(info)), "conv_schedule")
    assert info.cluster == 1 and info.pingpong == 1
    for bad in ("3x3", "2x", "x2", "21"):
        L.set_option("YB_CONV_MCAST", bad)
        assert L.lib.yb_conv_schedule(C.byref(d), 0, 0, 0, SMS, C.byref(info)) != 0
