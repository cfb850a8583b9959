"""CPU tests of the fp8 (e4m3) inference plan and of the e4m3 rounding used by the GPU tests (no device needed)."""
import ctypes as C

import torch

from tests import fp8_ref as F


def _lib():
    from yolov3_tensorflow_b200 import _lib
    return _lib


def _plan(L, dtype, training=0, n=2, h=416, w=416):
    h_ = C.c_void_p()
    rc = L.lib.yb_net_create(C.byref(h_), 80, n, h, w, dtype, training)
    return rc, h_


def test_e4m3_plan_host_only():
    """An e4m3 plan has the same 75 layers as the fp16 plan and a smaller activation arena (1-byte buffers after
    Conv_3)."""
    L = _lib()
    sizes = {}
    for dt in (L.YB_F16, L.YB_E4M3):
        rc, h = _plan(L, dt)
        assert rc == 0, L.lib.yb_last_error_string()
        try:
            assert L.lib.yb_net_num_layers(h) == 75
            a, p = C.c_size_t(), C.c_size_t()
            L.check(L.lib.yb_net_arena_bytes(h, C.byref(a), C.byref(p)), "arena_bytes")
            sizes[dt] = a.value
            for i in range(75):
                info = L.LayerInfo()
                L.check(L.lib.yb_net_layer_info(h, i, C.byref(info)), "layer_info")
                assert info.index == i
        finally:
            L.lib.yb_net_destroy(h)
    assert sizes[L.YB_E4M3] < 0.7 * sizes[L.YB_F16], sizes   # layers 0-2 keep their large fp16 buffers


def test_e4m3_training_rejected():
    L = _lib()
    rc, h = _plan(L, L.YB_E4M3, training=1)
    assert rc == -1 and not h.value
    assert b"inference" in L.lib.yb_last_error_string()


def test_e4m3_round_matches_torch():
    """The reference rounding equals torch.float8_e4m3fn on every finite code and on every midpoint between two
    neighbouring codes (ties to even), and saturates at +-448."""
    codes = torch.arange(256, dtype=torch.int32).to(torch.uint8)
    vals = codes.view(torch.float8_e4m3fn).double()
    vals = vals[torch.isfinite(vals)]
    assert vals.numel() == 254                                 # 0x7f / 0xff are NaN
    torch.testing.assert_close(F.e4m3_round(vals), vals, rtol=0, atol=0)
    pos = torch.unique(vals[vals >= 0])
    mids = torch.cat([(pos[1:] + pos[:-1]) / 2, -(pos[1:] + pos[:-1]) / 2])
    want = mids.float().to(torch.float8_e4m3fn).double()       # midpoints are exact in float32
    torch.testing.assert_close(F.e4m3_round(mids), want, rtol=0, atol=0)
    big = torch.tensor([448.0, 460.0, 1e6, -500.0], dtype=torch.float64)
    clamped = big.clamp(-448, 448).float().to(torch.float8_e4m3fn).double()
    torch.testing.assert_close(F.e4m3_round(big), clamped, rtol=0, atol=0)
    # and the spacing helper: one ulp up from every positive finite value below 448 is the next code
    up = pos[:-1] + F.e4m3_ulp(pos[:-1])
    torch.testing.assert_close(up, pos[1:], rtol=0, atol=0)
