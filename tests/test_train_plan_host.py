"""CPU tests of the training-plan model in tests/train_plan_ref.py, on unbound training plans (no GPU needed): the
input-gradient routing table against yb_net_layer_info / yb_net_layer_schedule, and, through yb_conv_schedule on the
reconstructed requests, that every configuration of tests/test_gpu_train_plan.py has a kernel for each of its launches
and reaches what it exists for."""
import ctypes as C

import pytest

from tests import train_plan_ref as T


@pytest.fixture
def L():
    from yolov3_tensorflow_b200 import _lib
    T.set_options(_lib, {})
    yield _lib
    T.set_options(_lib, {})


def _infos(L, n, H, W, code):
    net = C.c_void_p()
    L.check(L.lib.yb_net_create(C.byref(net), T.CLASSES, n, H, W, code, 1), "net_create")
    try:
        rows = []
        for i in range(L.lib.yb_net_num_layers(net)):
            info, s = L.LayerInfo(), L.LayerSchedule()
            L.check(L.lib.yb_net_layer_info(net, i, C.byref(info)), "layer_info")
            L.check(L.lib.yb_net_layer_schedule(net, i, T.SMS, C.byref(s)), "layer_schedule")
            rows.append((info, s))
        return rows
    finally:
        L.lib.yb_net_destroy(net)


def test_routing_table(L):
    topo = T.Topology()
    rows = _infos(L, 2, 416, 416, L.YB_BF16)
    assert len(rows) == len(topo.table) == 75
    assert [info.index for info, s in rows if s.residual] == topo.residual
    assert [info.index for info, _ in rows if info.upsample2x] == topo.upsample
    assert [info.index for info, _ in rows if not info.has_bn] == topo.heads
    routes = {i: topo.route(i) for i in range(1, 75)}
    assert {i for i, r in routes.items() if r[0] == "inplace"} == {26, 43, 57, 65}
    assert {i: r[1] for i, r in routes.items() if r[0] == "pass"} == {b - 1: b for b in topo.residual}
    # the shortcut of layers 25 and 42 lives in a concat buffer: dA(out_b) has a wider row pitch than the dgrad output
    assert (topo.out_ld[25], topo.in_ld(24), topo.out_off[25]) == (384, 256, 128)
    assert (topo.out_ld[42], topo.in_ld(41), topo.out_off[42]) == (768, 512, 256)
    for i in range(1, 75):
        info = rows[i][0]
        assert info.cin == sum(rows[j][0].cout for j in topo.inputs[i]), i
        for j in topo.inputs[i]:
            up = 2 if rows[j][0].upsample2x else 1
            assert (rows[j][0].out_h * up, rows[j][0].out_w * up) == (info.in_h, info.in_w), (i, j)
        if len(topo.inputs[i]) == 1:
            assert topo.in_ld(i) - topo.out_off[topo.inputs[i][0]] >= info.cin


@pytest.mark.parametrize("cid,opts,dt,n,hw", T.CONFIGS, ids=[c[0] for c in T.CONFIGS])
def test_configuration_premise(L, cid, opts, dt, n, hw):
    """Every launch of the configuration has a kernel, and the configuration reaches what it exists for."""
    T.set_options(L, opts)
    code = L.YB_F16 if dt == "fp16" else L.YB_BF16
    topo = T.Topology()
    infos = [info for info, _ in _infos(L, n, hw[0], hw[1], code)]
    scheds = T.schedules(L, topo, infos, n, code, "YB_DGRAD_S2" in opts)
    T.premise(cid, scheds, topo)
    if cid == "reg+mcast":
        # the register epilogue makes the dgrads cooperative: some of them run ping-pong without it
        T.set_options(L, {"YB_CONV_MCAST": "2x2"})
        plain = T.schedules(L, topo, infos, n, code, False)
        assert any(p[5].pingpong and not r[5].pingpong for i in scheds for p, r in zip(plain[i], scheds[i])
                   if r[0].startswith("dgrad"))


def test_schedule_rejects_unknown_option_value(L):
    """A configuration the library cannot run fails with its message, at selection time (and so when a plan binds)."""
    topo = T.Topology()
    infos = [info for info, _ in _infos(L, 2, 416, 416, L.YB_BF16)]
    L.set_option("YB_CONV_MCAST", "3x3")
    with pytest.raises(AssertionError, match="YB_CONV_MCAST must be 0, 2x1, 1x2 or 2x2"):
        T.schedules(L, topo, infos, 2, L.YB_BF16, False)
