"""The TMA-store epilogue of the implicit-GEMM conv (csrc/conv_igemm.cu, epilogue_tma, YB_CONV_EPI) on the GPU.

With YB_CONV_EPI=tma every warp keeps its accumulator fragments in registers, applies scale / shift, leaky and the
residual there, packs to 16 bits, writes a 16-row x 64-column swizzled slab with stmatrix and stores it by TMA; with
stage the values go through the fp32 staging tile.  Both do the same operations in the same order, so every output
must be byte-identical between the two and within the float64 bound of tests/conv_ref.py.  Sentinels around the output
(guard rows before and after, the columns outside a channel slice) must survive: the TMA clips rows >= M and columns
>= cout.  Requests the TMA store cannot serve (statistics, fp32 output, 2x upsample, the dgrad parity scatter, e4m3)
must report and run the staged epilogue under YB_CONV_EPI=tma."""
import ctypes as C

import pytest
import torch

from tests import conv_ref as R
from tests.test_gpu_conv_schedule import GUARD, FwdCase, _guards

pytestmark = pytest.mark.gpu

KEYS = ("YB_CONV_EPI", "YB_CONV_RES", "YB_CONV_MCAST", "YB_CONV_PP", "YB_CONV_CTAS", "YB_CONV_EG", "YB_CONV_MODE",
        "YB_CONV_MC")
DT = (torch.float16, torch.bfloat16)
_dt_id = {torch.float16: "f16", torch.bfloat16: "bf16"}


@pytest.fixture
def L():
    from yolov3_tensorflow_b200 import _lib
    for k in KEYS:
        _lib.set_option(k, None)
    yield _lib
    for k in KEYS:
        _lib.set_option(k, None)


def _schedule(L, d, kh=0, kw=0, stats=False):
    s = C.c_int()
    L.check(L.lib.yb_device_info(C.byref(s), None, None), "device_info")
    info = L.ConvSchedule()
    L.check(L.lib.yb_conv_schedule(C.byref(d), kh, kw, int(stats), s.value, C.byref(info)), "conv_schedule")
    return info


def _epi_ab(L, name, case, pp=None, mcast=None, cap=None, res=None, min_upw=0, want=None):
    """The case with YB_CONV_EPI=stage (checked against float64), then with tma: byte-identical outputs.  want: the
    (pingpong, block_n, block_k) the case is about."""
    for key, val in (("YB_CONV_PP", pp), ("YB_CONV_MCAST", mcast), ("YB_CONV_CTAS", cap), ("YB_CONV_RES", res)):
        L.set_option(key, val)
    outs = {}
    for mode in ("stage", "tma"):
        L.set_option("YB_CONV_EPI", mode)
        i = _schedule(L, case.desc)
        if want is not None:
            assert (i.pingpong, i.block_n, i.block_k) == want, f"{name}: schedule {(i.pingpong, i.block_n, i.block_k)}"
        if mcast not in (None, "0") and i.pingpong:
            assert i.cluster > 1, f"{name}: no cluster under {mcast}"
        if case.res_mode is not None:
            assert i.res_smem == (res != "ldg" and i.pingpong == 1 and i.block_n == 128 and i.block_k == 64), name
        # (a residual that is not prefetched into shared memory keeps the staged epilogue: yb_conv_schedule's epi_tma
        # describes the launch without a residual or with a prefetched one)
        assert i.epi_tma == (mode == "tma"), f"{name} {mode}: epilogue"
        upw = R.units_per_warpgroup(i)
        assert upw >= min_upw, f"{name}: only {upw} units per warpgroup"
        buf, ssum, ssq = case.run()
        if mode == "stage":
            outs[mode], worst = case.check(f"{name} stage", buf, ssum, ssq, upw, i.grid)
        else:
            _guards(f"{name} tma", buf, case.rows, case.out_off, case.cout)
            outs[mode] = buf[GUARD:GUARD + case.rows, case.out_off:case.out_off + case.cout].clone()
            R.check_out(outs[mode], case.ref, case.bound, f"{name} tma")
            print(f"EPI {name} pp={i.pingpong} mcast={mcast} cap={cap} res={res}: cluster {i.cluster} grid {i.grid} "
                  f"units/wg {upw} worst {worst:.3f}")
    assert torch.equal(outs["stage"].view(torch.int16), outs["tma"].view(torch.int16)), \
        f"{name} pp={pp} mcast={mcast} cap={cap} res={res}: the TMA-store epilogue changed the output bits"


# (k, stride, cin, cout, leaky) -> (pingpong, block_n, block_k) by the shape rule: 64- and 128-column tiles, 64- and
# 128-byte k-block rows, 1x1 and 3x3, stride 2, leaky on and off.  3 x 20 x 20 = 1200 pixels = 9.4 m-tiles (stride 2:
# 300 = 2.3): the last tile is partial, and under 2 x 1 / 2 x 2 clusters the last cluster has a rank wholly past M.
SHAPES = {
    "1x1_bn64_k64": ((1, 1, 128, 64, True), (1, 64, 64)),
    "1x1_bn64_k32": ((1, 1, 96, 32, False), (1, 64, 32)),
    "1x1_bn128_k64_coop": ((1, 1, 256, 128, True), (0, 128, 64)),
    "1x1_bn128_k32_coop": ((1, 1, 32, 256, True), (0, 128, 32)),
    "3x3_bn128_k64": ((3, 1, 64, 128, True), (1, 128, 64)),
    "3x3_bn128_k32": ((3, 1, 32, 128, False), (1, 128, 32)),
    "3x3_bn64_k64": ((3, 1, 64, 192, True), (1, 64, 64)),
    "3x3_s2_bn128": ((3, 2, 64, 256, True), (1, 128, 64)),
    "1x1_cout96_coop": ((1, 1, 64, 96, True), (0, 128, 64)),      # the second 64-column box: 32 valid columns
}


@pytest.mark.parametrize("dtype", DT, ids=_dt_id.get)
@pytest.mark.parametrize("name", list(SHAPES))
def test_epi_shapes_bit_identical(L, name, dtype):
    (k, s, cin, cout, leaky), want = SHAPES[name]
    case = FwdCase(L, 3, 20, 20, cin, cout, k, s, dtype=dtype, leaky=leaky, seed=list(SHAPES).index(name) + 70)
    _epi_ab(L, name, case, want=want)
    if want[0]:
        for mcast in ("2x1", "2x2"):
            _epi_ab(L, name, case, mcast=mcast)
        _epi_ab(L, name, case, pp="0")               # the same tiles under the cooperative schedule
    else:
        _epi_ab(L, name, case, pp="1")               # ... and under ping-pong


@pytest.mark.parametrize("dtype", DT, ids=_dt_id.get)
def test_epi_cooperative_clusters(L, dtype):
    """YB_CONV_MODE=2cta: the cooperative 2 x 1 and 4 x 1 clusters."""
    case = FwdCase(L, 3, 20, 20, 128, 256, 1, 1, dtype=dtype, seed=80)
    L.set_option("YB_CONV_MODE", "2cta")
    _epi_ab(L, "coop 2x1", case, want=(0, 128, 64))
    L.set_option("YB_CONV_MC", "1")
    _epi_ab(L, "coop 4x1", case, want=(0, 128, 64))


@pytest.mark.parametrize("dtype", DT, ids=_dt_id.get)
def test_epi_channel_slice(L, dtype):
    """The output is a channel slice of a wider buffer (out_ld > cout, offset base), as the concat buffers of the plan:
    64- and 128-column tiles, and an input slice as well."""
    for k, cin, cout in ((1, 128, 64), (3, 64, 128), (1, 256, 128)):
        case = FwdCase(L, 3, 20, 20, cin, cout, k, 1, dtype=dtype, in_extra=32, out_extra=192, seed=81 + k)
        assert case.out_off > 0 and case.out_ld > cout
        _epi_ab(L, f"slice k{k} cout{cout}", case)
        _epi_ab(L, f"slice k{k} cout{cout}", case, cap="2", min_upw=2)


@pytest.mark.parametrize("dtype", DT, ids=_dt_id.get)
@pytest.mark.parametrize("res", ("smem", "ldg"))
def test_epi_residual(L, res, dtype):
    """A residual through the shared-memory shortcut tile (added in place, stored from there), and from global memory
    (YB_CONV_RES=ldg, 64-column tiles), which keeps the staged epilogue;
    separate and in place in a buffer of row pitch cout + 64 (res_ld > cout); 1200 pixels: partial last tile, idle
    cluster ranks; capped grids: every warpgroup reuses its shortcut tile several times."""
    sep = FwdCase(L, 3, 20, 20, 192, 256, 3, 1, dtype=dtype, res="sep", seed=85)
    inplace = FwdCase(L, 3, 20, 20, 128, 256, 3, 1, dtype=dtype, res="inplace", out_extra=64, seed=86)
    assert inplace.desc.res_ld > inplace.desc.cout
    for name, case in (("res sep", sep), ("res inplace", inplace)):
        for mcast, cap, upw in (("0", None, 0), ("2x1", None, 0), ("2x2", None, 0), ("0", "1", 4), ("0", "2", 4),
                                ("2x2", "4", 2)):
            _epi_ab(L, name, case, mcast=mcast, cap=cap, res=res, min_upw=upw)
    small = FwdCase(L, 3, 20, 20, 128, 64, 1, 1, dtype=dtype, res="sep", seed=87)   # 64-column tiles: no shortcut tile
    _epi_ab(L, "res bn64", small, res=res)


@pytest.mark.parametrize("dtype", DT, ids=_dt_id.get)
def test_epi_buffer_reuse_many_units(L, dtype):
    """2 x 104 x 104 pixels = 169 m-tiles on one or two CTAs / one cluster: every warp rewrites its output slab (its
    rows of the shortcut tile) 40-170 times, so a slab rewritten before its store had been read shows as a wrong tile."""
    plain = FwdCase(L, 2, 104, 104, 64, 128, 3, 1, dtype=dtype, seed=88)
    narrow = FwdCase(L, 2, 104, 104, 128, 64, 1, 1, dtype=dtype, seed=89)
    wide1 = FwdCase(L, 2, 104, 104, 64, 128, 1, 1, dtype=dtype, seed=90)
    resid = FwdCase(L, 2, 104, 104, 64, 128, 3, 1, dtype=dtype, res="sep", seed=91)
    for name, case in (("reuse 3x3", plain), ("reuse 1x1 bn64", narrow), ("reuse 1x1 coop", wide1), ("reuse res", resid)):
        for mcast, cap in (("0", "1"), ("0", "2"), ("2x2", "4")):
            _epi_ab(L, name, case, mcast=mcast, cap=cap, min_upw=20)


def test_epi_ineligible_requests_run_staged(L):
    """Statistics, fp32 output, 2x upsample, the dgrad parity scatter and e4m3 keep the staged epilogue under
    YB_CONV_EPI=tma: reported so, and the outputs are right."""
    L.set_option("YB_CONV_EPI", "tma")
    for name, kw in (("stats", dict(stats=True)), ("fp32", dict(out_fp32=True)), ("upsample", dict(upsample=True))):
        case = FwdCase(L, 2, 26, 26, 128, 255 if name == "fp32" else 128, 1, 1, seed=92, **kw)
        i = _schedule(L, case.desc, stats=case.stats)
        assert i.epi_tma == 0, name
        buf, ssum, ssq = case.run()
        case.check(f"ineligible {name}", buf, ssum, ssq, R.units_per_warpgroup(i), i.grid)
    d = L.ConvDesc(n=2, h=26, w=26, cin=128, cout=64, ksize=1, stride=1, in_ld=128, out_ld=64, res_ld=0, dtype=L.YB_F16,
                   out_fp32=0, leaky=0, upsample2x=0)
    assert _schedule(L, d, kh=2, kw=2).epi_tma == 0, "dgrad parity class"
    assert _schedule(L, d).epi_tma == 1
    d.dtype = L.YB_E4M3
    assert _schedule(L, d).epi_tma == 0, "e4m3"


def test_epi_e4m3_runs_staged(L):
    """An e4m3 conv under YB_CONV_EPI=tma runs (the staged epilogue) and gives the bytes it gives without the option."""
    from tests import test_gpu_fp8 as F8
    c = F8.Case("1x1 256->128", 2, 18, 14, 256, 128)
    t = F8._setup(L, c, seed=3)
    outs = []
    for mode in (None, "tma"):
        L.set_option("YB_CONV_EPI", mode)
        outs.append(F8._run(L, c, t))
    assert bool((outs[0][F8.GUARD:F8.GUARD + t["M"]] != F8.SENT).any()), "nothing written"
    assert torch.equal(outs[0], outs[1])
