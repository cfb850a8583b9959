"""CPU tests of the conv test machinery and of the conv kernel selection.

- The float64 checker of tests/conv_ref.py rejects outputs with the faults a work-unit schedule can make, and accepts
  the correctly rounded output.
- yb_conv_schedule (host-only) reports the kernel and grid every layer of the 80-class plan gets, and the YB_CONV_PP /
  YB_CONV_CTAS switches change exactly what DESIGN.md §5b says they change."""
import ctypes as C
import os

import pytest
import torch

from tests import conv_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "yolov3_tensorflow_b200", "libyolob200.so")

FAULTS = ["k-block missing", "halves swapped", "tail row from neighbour tile", "leaky slope 0.125",
          "tile missing from statistics", "residual added twice", "round toward zero"]


def _rtz(v32, dtype):
    """fp32 -> dtype rounded toward zero."""
    rn = v32.to(dtype)
    bits = rn.view(torch.int16)
    up = rn.float().abs() > v32.abs()           # round-to-nearest went away from zero: one ulp back (sign-magnitude)
    return torch.where(up, bits - 1, bits).view(dtype)


def _faults(dtype):
    """Small 1x1 conv (M = 200: one full 128-row tile and a 72-row tail; K = 128 = two 64-channel k-blocks) with its
    float64 reference, the correctly rounded kernel output, and the seven faulty ones."""
    g = torch.Generator().manual_seed(21)
    n, h, w, cin, cout = 2, 10, 10, 128, 64
    x = torch.randn((n, h, w, cin), generator=g).to(dtype)
    wt = (torch.randn((cout, 1, 1, cin), generator=g) / cin ** 0.5).to(dtype)
    scale = torch.rand(cout, generator=g) + 0.5
    shift = torch.randn(cout, generator=g) * 0.1
    res = torch.randn((n * h * w, cout), generator=g).to(dtype)
    raw, S = R.conv_raw(x, wt, 1, 0)
    ref = R.epilogue(raw, scale, shift, True, res)
    n16 = cin // 16

    def store(raw_, slope=R.SLOPE, res_=res, rtz=False):
        v = raw_.float() * scale + shift                      # fp32 epilogue (the raw sums are exact enough here)
        v = torch.where(v > 0, v, slope * v) + res_.float()
        return _rtz(v, dtype) if rtz else v.to(dtype)

    good = store(raw)
    cols = x.double().reshape(-1, cin)
    wm = wt.double().reshape(cout, cin)
    bad = {}
    r = raw.clone(); r[64:128] -= cols[64:128, 64:128] @ wm[:, 64:128].t()
    bad["k-block missing"] = store(r)
    o = good.clone(); o[0:64], o[64:128] = good[64:128].clone(), good[0:64].clone()
    bad["halves swapped"] = o
    o = good.clone(); o[199] = good[199 - 128]
    bad["tail row from neighbour tile"] = o
    bad["leaky slope 0.125"] = store(raw, slope=0.125)
    rr = res.clone().float(); rr[128:200, 32:64] *= 2
    bad["residual added twice"] = store(raw, res_=rr)
    bad["round toward zero"] = store(raw, rtz=True)
    return raw, S, ref, n16, scale, shift, res, good, bad


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_checker_rejects_schedule_faults(dtype):
    """Every simulated fault is rejected by the per-element bound and the statistics bound; the correctly rounded
    output and the fp32 statistics pass.  The old criterion (|err| <= 2^-9 max(1, |ref|) for fp16, 2^-6 for bf16) lets
    the round-toward-zero store through in both types, since one ulp of fp16 (bf16) is 2^-10 (2^-7) relative."""
    raw, S, ref, n16, scale, shift, res, good, bad = _faults(dtype)
    bound = R.out_bound(ref, S, n16, dtype, scale, shift, res)
    assert R.check_out(good, ref, bound, "correct output") <= 1.0
    old_misses = []
    for name, got in bad.items():
        with pytest.raises(AssertionError):
            R.check_out(got, ref, bound, name)
        if R.old_criterion_ok(got, ref, dtype):
            old_misses.append(name)
    assert old_misses == ["round toward zero"]
    # statistics: fp32 sums of the fp32 accumulators pass; one 128-row tile left out of one n-tile's sums does not
    depth = R.stats_depth(units_per_wg=1, grid=1)
    b_sum, b_sq = R.stats_bound(raw, S, n16, depth)
    r32 = raw.float()
    s_ok, q_ok = r32.sum(0), (r32 * r32).sum(0)
    assert bool(((s_ok.double() - raw.sum(0)).abs() <= b_sum).all())
    assert bool(((q_ok.double() - (raw * raw).sum(0)).abs() <= b_sq).all())
    s_bad = s_ok - r32[0:128].sum(0)
    q_bad = q_ok - (r32[0:128] ** 2).sum(0)
    assert not bool(((s_bad.double() - raw.sum(0)).abs() <= b_sum).all())
    assert not bool(((q_bad.double() - (raw * raw).sum(0)).abs() <= b_sq).all())
    assert set(bad) | {"tile missing from statistics"} == set(FAULTS)


def test_ulp_spacing():
    a = torch.tensor([1.0, 1.5, 2.0, 0.0, 2.0 ** -20, 65504.0], dtype=torch.float64)
    assert R.ulp(a, torch.float16).tolist() == [2.0 ** -10, 2.0 ** -10, 2.0 ** -9, 2.0 ** -24, 2.0 ** -24, 32.0]
    assert R.ulp(a[:3], torch.bfloat16).tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -6]
    assert R.ulp(torch.tensor([0.0], dtype=torch.float64), torch.bfloat16).item() == 2.0 ** -133


# ------------------------------------------------------------------------- kernel selection of the 80-class plan
@pytest.fixture(scope="module")
def L():
    if not os.path.exists(LIB):
        import __graft_entry__ as g
        g.build()
    from yolov3_tensorflow_b200 import _lib
    return _lib


@pytest.fixture
def opts(L):
    keys = ("YB_CONV_PP", "YB_CONV_CTAS", "YB_CONV_EG", "YB_CONV_MODE", "YB_CONV_MC", "YB_CONV_EPI")
    for k in keys:
        L.set_option(k, None)
    yield lambda **kw: [L.set_option(k, v) for k, v in kw.items()]
    for k in keys:
        L.set_option(k, None)


SMS = 132


def _sched(L, d, kh=0, kw=0, stats=0, sms=SMS):
    info = L.ConvSchedule()
    L.check(L.lib.yb_conv_schedule(C.byref(d), kh, kw, stats, sms, C.byref(info)), "conv_schedule")
    return info


def _plan_convs(L, n, training):
    """(name, desc, kh, kw, with_stats) of every implicit-GEMM conv the 80-class plan at 416^2 can run: the forward of
    layers 1..74 and, for training, their dgrad (stride 1: a conv over dz; stride 2: the four parity classes)."""
    h = C.c_void_p()
    L.check(L.lib.yb_net_create(C.byref(h), 80, n, 416, 416, 0, 1 if training else 0), "net_create")
    out = []
    try:
        for i in range(1, L.lib.yb_net_num_layers(h)):
            li = L.LayerInfo()
            L.check(L.lib.yb_net_layer_info(h, i, C.byref(li)), "layer_info")
            head = not li.has_bn
            d = L.ConvDesc(n=n, h=li.in_h, w=li.in_w, cin=li.cin, cout=li.cout, ksize=li.ksize, stride=li.stride,
                           in_ld=li.cin, out_ld=li.cout, res_ld=0, dtype=L.YB_F16, out_fp32=int(head), leaky=int(not head),
                           upsample2x=li.upsample2x)
            out.append((f"fwd{i}", d, 0, 0, int(training and not head)))
            if not training:
                continue
            kco = (li.cout + 31) // 32 * 32
            if li.stride == 1:
                dd = L.ConvDesc(n=n, h=li.in_h, w=li.in_w, cin=kco, cout=li.cin, ksize=li.ksize, stride=1, in_ld=kco,
                                out_ld=li.cin, res_ld=li.cin, dtype=L.YB_F16, out_fp32=0, leaky=0, upsample2x=0)
                out.append((f"dgrad{i}", dd, 0, 0, 0))
            else:
                dd = L.ConvDesc(n=n, h=li.out_h, w=li.out_w, cin=kco, cout=li.cin, ksize=1, stride=1, in_ld=kco,
                                out_ld=li.cin, res_ld=li.cin, dtype=L.YB_F16, out_fp32=0, leaky=0, upsample2x=0)
                for c in range(4):
                    out.append((f"dgrad{i}.{c}", dd, 1 + (c >> 1), 1 + (c & 1), 0))
    finally:
        L.lib.yb_net_destroy(h)
    return out


def _expected_stages(bm, bn, bk):
    return min(8, 196 * 1024 // ((bm + bn) * bk * 2))


@pytest.mark.parametrize("n,training", [(64, False), (32, True)])
def test_plan_schedule_table(L, opts, n, training):
    convs = _plan_convs(L, n, training)
    assert len(convs) == (74 if not training else 74 + 74 + 3 * 5)      # five stride-2 layers: 4 classes each
    for name, d, kh, kw, st in convs:
        opts()
        i = _sched(L, d, kh, kw, st)
        windowed = d.ksize * d.ksize > 1 or kh * kw > 1
        assert (i.consumers, i.cluster, i.block_m) == (2, 1, 128), name
        assert i.block_n == (128 if (d.cout + 63) // 64 * 64 % 128 == 0 else 64), name
        assert i.block_k == (64 if d.cin % 64 == 0 else 32), name
        # default rule: windowed convs and 64-column 1x1 convs ping-pong, 128-column 1x1 convs cooperative
        assert i.pingpong == int(windowed or i.block_n == 64), name
        assert i.stages == (6 if (i.block_n, i.block_k) == (128, 64) else 8), name
        assert i.stages == _expected_stages(i.block_m, i.block_n, i.block_k), name
        taps = (d.ksize * d.ksize) if kh == 0 else kh * kw
        assert i.num_kb == taps * d.cin // i.block_k, name
        P, Q = d.h // d.stride, d.w // d.stride
        assert i.num_m_tiles == -(-n * P * Q // 128) and i.num_n_tiles == (d.cout + 63) // 64 * 64 // i.block_n, name
        assert i.grid == min(i.num_m_tiles * i.num_n_tiles, SMS), name
        # YB_CONV_PP: 0 = cooperative everywhere, 1 = ping-pong everywhere the kernel allows
        for v in ("0", "1"):
            opts(YB_CONV_PP=v)
            j = _sched(L, d, kh, kw, st)
            assert j.pingpong == int(v) and (j.consumers, j.cluster, j.stages, j.num_kb, j.grid) == \
                (2, 1, i.stages, i.num_kb, i.grid), (name, v)
        # clusters, one consumer warpgroup and the register epilogue are cooperative whatever YB_CONV_PP says
        for kw_ in ({"YB_CONV_MODE": "2cta"}, {"YB_CONV_MODE": "2cta", "YB_CONV_MC": "1"}, {"YB_CONV_EG": "1"},
                    {"YB_CONV_EPI": "reg"}):
            for v in (None, "1"):
                opts(YB_CONV_MODE=None, YB_CONV_MC=None, YB_CONV_EG=None, YB_CONV_EPI=None)
                opts(YB_CONV_PP=v, **kw_)
                j = _sched(L, d, kh, kw, st)
                if "YB_CONV_EPI" in kw_ and st:          # no register epilogue with statistics: the default kernel
                    assert j.pingpong == (1 if v == "1" else i.pingpong), (name, kw_, v)
                    continue
                assert j.pingpong == 0, (name, kw_, v)
                if "YB_CONV_EG" in kw_:
                    assert (j.consumers, j.block_m) == (1, 64), name
                    assert j.stages == _expected_stages(64, j.block_n, j.block_k), name
                if "YB_CONV_MODE" in kw_:
                    cs = 4 if "YB_CONV_MC" in kw_ else 2
                    assert j.cluster == cs and j.grid % cs == 0, name
        opts(YB_CONV_PP=None, YB_CONV_MODE=None, YB_CONV_MC=None, YB_CONV_EG=None, YB_CONV_EPI=None)
        # YB_CONV_CTAS: the grid only
        for cap in (1, 2, 3, 7, 1000):
            opts(YB_CONV_CTAS=str(cap))
            j = _sched(L, d, kh, kw, st)
            assert j.grid == min(cap, i.num_m_tiles * i.num_n_tiles, SMS), (name, cap)
            assert (j.pingpong, j.num_kb, j.stages, j.num_m_tiles) == (i.pingpong, i.num_kb, i.stages, i.num_m_tiles)
        opts(YB_CONV_CTAS=None)


def test_ctas_cap_whole_clusters(L, opts):
    d = L.ConvDesc(n=8, h=52, w=52, cin=64, cout=128, ksize=3, stride=1, in_ld=64, out_ld=128, res_ld=0, dtype=L.YB_F16,
                   out_fp32=0, leaky=1, upsample2x=0)
    units = -(-8 * 52 * 52 // 128)
    for mc, cs in ((None, 2), ("1", 4)):
        for cap, want in ((1, cs), (cs - 1, cs), (7, 7 // cs * cs), (None, SMS // cs * cs)):
            opts(YB_CONV_MODE="2cta", YB_CONV_MC=mc, YB_CONV_CTAS=None if cap is None else str(cap))
            j = _sched(L, d)
            assert j.cluster == cs and j.grid == want, (cs, cap, j.grid)
    opts(YB_CONV_MODE=None, YB_CONV_MC=None, YB_CONV_CTAS="5")
    assert _sched(L, d).grid == 5 and _sched(L, d, sms=4).grid == 4
    opts(YB_CONV_CTAS=None)
    assert _sched(L, d, sms=100).grid == 100 and units > 132


def test_schedule_rejects_bad_arguments(L, opts):
    d = L.ConvDesc(n=1, h=8, w=8, cin=24, cout=64, ksize=3, stride=1, in_ld=24, out_ld=64, res_ld=0, dtype=0,
                   out_fp32=0, leaky=1, upsample2x=0)
    info = L.ConvSchedule()
    assert L.lib.yb_conv_schedule(C.byref(d), 0, 0, 0, SMS, C.byref(info)) == -1
    assert b"cin" in L.lib.yb_last_error_string()
    d.cin = d.in_ld = 64
    assert L.lib.yb_conv_schedule(C.byref(d), 0, 0, 0, 0, C.byref(info)) == -1
    assert L.lib.yb_conv_schedule(C.byref(d), 3, 1, 0, SMS, C.byref(info)) == -1
    assert L.lib.yb_conv_schedule(C.byref(d), 0, 0, 0, SMS, C.byref(info)) == 0
