"""CPU tests: which launches take the TMA-store epilogue of the implicit-GEMM conv (yb_net_layer_schedule on unbound
plans, yb_conv_schedule) and the YB_CONV_EPI option.  No GPU needed."""
import ctypes as C

import pytest

KEYS = ("YB_CONV_EPI", "YB_CONV_RES", "YB_CONV_MCAST", "YB_CONV_PP", "YB_CONV_CTAS", "YB_CONV_EG", "YB_CONV_MODE",
        "YB_CONV_MC", "YB_HALO")
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


@pytest.mark.parametrize("dtype", ("f16", "bf16"))
def test_plan_epilogue_table(L, dtype):
    """The batch-64 16-bit inference plan stores by TMA from exactly its plain 16-bit implicit-GEMM layers: not the
    three fp32 detection heads, not the two 2x-upsampling convs, not the halo-kernel layers."""
    rows = _plan_table(L, L.YB_F16 if dtype == "f16" else L.YB_BF16)
    want = [info.index for info, s in rows if s.igemm and info.has_bn and not info.upsample2x]
    assert len(want) == 67 and len([1 for _, s in rows if s.igemm]) == 72
    assert [info.index for info, s in rows if s.epi_tma] == want
    # both schedules and every cluster shape of the plan are among them
    assert {(s.pingpong, s.cluster_m, s.cluster_n) for _, s in rows if s.epi_tma} >= {(1, 1, 1), (1, 2, 1), (1, 2, 2)}


def test_plan_epilogue_option_and_other_plans(L):
    """YB_CONV_EPI=stage: nowhere; training and e4m3 plans: nowhere.  Under YB_CONV_EPI=tma the e4m3 plan takes it only
    for Conv_2, its one fp16 implicit-GEMM layer."""
    L.set_option("YB_CONV_EPI", "stage")
    assert not any(s.epi_tma for _, s in _plan_table(L, L.YB_F16))
    L.set_option("YB_CONV_EPI", None)
    assert not any(s.epi_tma for _, s in _plan_table(L, L.YB_BF16, training=1, n=32))
    assert not any(s.epi_tma for _, s in _plan_table(L, L.YB_E4M3))
    L.set_option("YB_CONV_EPI", "tma")
    assert [info.index for info, s in _plan_table(L, L.YB_E4M3) if s.epi_tma] == [2]


def _conv_schedule(L, kh=0, kw=0, stats=0, **kw_):
    d = dict(n=8, h=52, w=52, cin=128, cout=256, ksize=3, stride=1, in_ld=128, out_ld=256, res_ld=256,
             dtype=L.YB_F16, out_fp32=0, leaky=1, upsample2x=0)
    d.update(kw_)
    desc = L.ConvDesc(**d)
    info = L.ConvSchedule()
    rc = L.lib.yb_conv_schedule(C.byref(desc), kh, kw, stats, SMS, C.byref(info))
    return rc, info


def test_conv_schedule_reports_the_epilogue(L):
    rc, i = _conv_schedule(L)
    assert rc == 0 and i.epi_tma == 0, "a single conv keeps the staged epilogue unless asked"
    L.set_option("YB_CONV_EPI", "tma")
    rc, i = _conv_schedule(L)
    assert rc == 0 and i.epi_tma == 1 and i.pingpong == 1
    assert (i.stages, i.res_stages, i.res_smem) == (6, 4, 1), "the ring depths do not depend on the epilogue"
    for kw in (dict(dtype=L.YB_BF16), dict(ksize=1, cin=256, in_ld=256), dict(cout=64, out_ld=64, res_ld=64),
               dict(cin=96, in_ld=96), dict(stride=2), dict(out_ld=768)):
        rc, i = _conv_schedule(L, **kw)
        assert rc == 0 and i.epi_tma == 1, kw
    for mcast in ("2x1", "1x2", "2x2"):
        L.set_option("YB_CONV_MCAST", mcast)
        rc, i = _conv_schedule(L)
        assert rc == 0 and i.epi_tma == 1 and i.cluster > 1, mcast
    L.set_option("YB_CONV_MCAST", None)
    L.set_option("YB_CONV_MODE", "2cta")
    rc, i = _conv_schedule(L)
    assert rc == 0 and i.epi_tma == 1 and i.pingpong == 0 and i.cluster == 2
    L.set_option("YB_CONV_MODE", None)
    # what the TMA store cannot serve keeps the staged epilogue: statistics, fp32 output, 2x upsample, the dgrad
    # parity classes, e4m3, one-warpgroup CTAs
    for kw in (dict(stats=1), dict(out_fp32=1, cout=255, ksize=1), dict(upsample2x=1, ksize=1), dict(kh=2, kw=1, ksize=1),
               dict(dtype=L.YB_E4M3)):
        rc, i = _conv_schedule(L, **kw)
        assert rc == 0 and i.epi_tma == 0, kw
    L.set_option("YB_CONV_EG", "1")
    rc, i = _conv_schedule(L)
    assert rc == 0 and i.epi_tma == 0 and i.consumers == 1
    L.set_option("YB_CONV_EG", None)
    L.set_option("YB_CONV_EPI", "reg")
    rc, i = _conv_schedule(L)
    assert rc == 0 and i.epi_tma == 0
    for bad in ("TMA", "smem", "1"):
        L.set_option("YB_CONV_EPI", bad)
        assert _conv_schedule(L)[0] != 0, bad
