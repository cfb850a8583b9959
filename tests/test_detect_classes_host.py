"""CPU tests: the tile width of the fused-decode detection heads at every class count (yb_net_layer_schedule's
det_block_n on unbound plans).  No GPU needed."""
import ctypes as C

import pytest

SMS = 132


def _head_tiles(L, cn, dtype):
    net = C.c_void_p()
    L.check(L.lib.yb_net_create(C.byref(net), cn, 2, 416, 416, dtype, 0), "net_create")
    try:
        tiles = []
        for i in range(L.lib.yb_net_num_layers(net)):
            info, s = L.LayerInfo(), L.LayerSchedule()
            L.check(L.lib.yb_net_layer_info(net, i, C.byref(info)), "layer_info")
            L.check(L.lib.yb_net_layer_schedule(net, i, SMS, C.byref(s)), "layer_schedule")
            if info.has_bn:
                assert s.det_block_n == 0, i
            else:
                tiles.append(s.det_block_n)
        return tiles
    finally:
        L.lib.yb_net_destroy(net)


@pytest.mark.parametrize("dtype", ("f16", "bf16", "e4m3"))
def test_head_tile_width_per_class_count(dtype):
    """3 (5 + C) columns on the narrowest of 64, 128, 256: C 1-16 -> 64, 17-37 -> 128, 38-80 -> 256; none above 80."""
    from yolov3_tensorflow_b200 import _lib as L
    code = {"f16": L.YB_F16, "bf16": L.YB_BF16, "e4m3": L.YB_E4M3}[dtype]
    for cn in range(1, 86):
        want = 64 if cn <= 16 else 128 if cn <= 37 else 256 if cn <= 80 else 0
        assert _head_tiles(L, cn, code) == [want] * 3, cn
