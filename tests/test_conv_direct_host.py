"""CPU tests of the direct conv kernels' test machinery (tests/direct_ref.py, tests/test_gpu_conv_direct.py).

- The halo and thin instantiation tables, written out here from halo_kernel_type (csrc/conv_halo.cu) and
  thin_kernel_type (csrc/conv_thin.cu): the halo table agrees with the host-only yb_conv3x3_halo_supported over a grid
  of descriptors, and every instantiation of both tables is launched by the GPU case table, so an instantiation added
  later fails here until it is tested.
- Each bound helper holds for a float32 emulation of the kernel's arithmetic in the kernel's order, and rejects outputs
  with the faults a direct conv can make: a tap dropped at an image border, a neighbouring channel's shift, a row
  taken from the next image, a tile missing from the batch sums."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest
import torch

from tests import conv_ref as R
from tests import direct_ref as D
from tests import test_gpu_conv_direct as G
from tests.wgrad_ref import _ETA, _U16

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "yolov3_tensorflow_b200", "libyolob200.so")
F16, BF16 = torch.float16, torch.bfloat16
SMS = 132

# (dtype, cin, cout, stride, fused stem, e4m3 output, residual box): halo_kernel_type
HALO_TABLE = {(dt, 32, 64, 2, True, False, False) for dt in (F16, BF16)} | \
             {(dt, 32, 64, 1, False, False, box) for dt in (F16, BF16) for box in (False, True)} | \
             {(F16, 32, 64, 1, False, True, box) for box in (False, True)} | \
             {(dt, ci, co, s, False, False, False) for dt in (F16, BF16)
              for ci, co, s in ((32, 64, 2), (32, 128, 1), (32, 128, 2), (64, 64, 1), (64, 64, 2), (64, 128, 1))}
# (dtype, cout, stride, stem, split operands): thin_kernel_type
THIN_TABLE = {(dt, 32, 1, True, split) for dt in (F16, BF16) for split in (False, True)} | \
             {(dt, co, s, False, False) for dt in (F16, BF16) for co in (32, 64) for s in (1, 2)}


@pytest.fixture(scope="module")
def L():
    if not os.path.exists(LIB):
        import __graft_entry__ as g
        g.build()
    from yolov3_tensorflow_b200 import _lib
    return _lib


# ------------------------------------------------------------------------------------------------ instantiation tables
def test_halo_table_matches_library(L):
    """yb_conv3x3_halo_supported (plain requests: no fused stem, 16-bit output) over cin x cout x stride x dtype, output
    widths that are and are not a multiple of the 8-pixel tile, and leading dimensions that are odd or too small."""
    n_ok = 0
    for dt, ci, co, s in itertools.product((F16, BF16), (32, 64, 96), (32, 64, 128, 256), (1, 2)):
        for wo, ld_in, ld_out in itertools.product((16, 20), (ci, ci + 8, ci + 3, ci - 8), (co, co + 16, co + 5)):
            d = L.ConvDesc(n=2, h=13 * s, w=wo * s, cin=ci, cout=co, ksize=3, stride=s, in_ld=ld_in, out_ld=ld_out,
                           res_ld=0, dtype=G._code(L, dt), out_fp32=0, leaky=1, upsample2x=0)
            shape_ok = wo % 8 == 0 and ld_in >= ci and ld_in % 8 == 0 and ld_out >= co and ld_out % 8 == 0
            want = shape_ok and (dt, ci, co, s, False, False, False) in HALO_TABLE
            assert L.lib.yb_conv3x3_halo_supported(C.byref(d)) == int(want), (dt, ci, co, s, wo, ld_in, ld_out)
            n_ok += want
    assert n_ok == 2 * 7 * 2 * 2                       # 7 plain instantiations per dtype, 2 x 2 good leading dimensions
    # the unsupported shapes of the inference plan: 256 -> 512 at 26 x 26, and 20 x 20 (20 % 8 != 0)
    for h, ci, co in ((26, 256, 512), (20, 64, 128)):
        d = L.ConvDesc(n=1, h=h, w=h, cin=ci, cout=co, ksize=3, stride=1, in_ld=ci, out_ld=co, res_ld=0, dtype=0,
                       out_fp32=0, leaky=1, upsample2x=0)
        assert L.lib.yb_conv3x3_halo_supported(C.byref(d)) == 0


def test_every_instantiation_has_gpu_cases():
    halo, thin = G.case_keys()
    assert HALO_TABLE - halo == set(), f"halo instantiations without a GPU case: {sorted(map(str, HALO_TABLE - halo))}"
    assert THIN_TABLE - thin == set(), f"thin instantiations without a GPU case: {sorted(map(str, THIN_TABLE - thin))}"
    assert halo <= HALO_TABLE and thin <= THIN_TABLE, "a GPU case selects an instantiation the tables do not list"
    for c in G.HALO_CASES:
        if c.deep:
            tiles = c.n * -(-(c.h // c.s) // 16) * (c.w // c.s // 8)
            assert tiles >= G.DEEP_TILES * SMS, c.name
        else:
            assert not c.name.endswith("-small") or ((c.h // c.s) % 16 and (c.h // c.s) % 2 and c.n >= 3), c.name


# ------------------------------------------------------------------------------------------------ emulations
def _f32(a):
    return a.astype(np.float32)


def _store(v32, dt):
    return torch.from_numpy(v32).to(dt).double()


def _fma(a, b, c):
    """float32 fmaf, emulated: the float64 product of two float32 values is exact, the sum rounds once in float64 and
    once to float32 (double rounding: at most an extra half ulp, inside the bounds' slack)."""
    return _f32(a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64))


def _epi(acc, sc, sh, leaky):
    v = _fma(acc, sc, sh)
    return np.maximum(v, _f32(np.float32(0.1) * v)) if leaky else v


def _mma_acc(cols, wm):
    """float32 accumulation of exact products in k order, rounding after every add (an mma.sync / wgmma k16 step adds
    its 16 products in at most 4 rounded groups; one rounding per product is a finer model of the same chain)."""
    acc = np.zeros((cols.shape[0], wm.shape[1]), np.float32)
    for k in range(cols.shape[1]):
        acc = _f32(acc.astype(np.float64) + np.outer(cols[:, k], wm[k]))
    return acc


def _case(seed, n=2, h=6, w=10, cin=3, cout=32):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((n, h, w, cin), generator=g)
    x[0, 0, :3] = torch.rand((3, cin), generator=g) * 2.0 ** -12          # fp16 remainders in the subnormal range
    wt = torch.randn((cout, 3, 3, cin), generator=g) * 0.2
    sc, sh = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.1
    return x, wt, sc, sh


def _drop_border_tap(cols, w, cin):
    """im2col rows [M, 9 cin] with tap (r, s) = (1, 0) zeroed for the output pixels in the image's last column: the
    in-image left neighbour's contribution lost at the right border."""
    cols = cols.copy()
    cols[np.arange(cols.shape[0]) % w == w - 1, 3 * cin:4 * cin] = 0
    return cols


def _faults(emulate, got, sh, n, h, w):
    """Known-wrong outputs [n h w, c] (float64) of an emulation emulate(drop, shift): (name, tensor)."""
    row = got.reshape(n, h, w, -1).clone()
    row[0, -1] = row[1, -1]                                                  # image 0's last row from image 1
    return [("tap dropped at the border", emulate(True, sh)),
            ("neighbouring channel's shift", emulate(False, torch.roll(sh, -1))),
            ("row from the next image", row.reshape(got.shape))]


def _assert_teeth(got, ref, bound, faults):
    R.check_out(got, ref, bound, "correct emulation")
    for name, bad in faults:
        with pytest.raises(AssertionError):
            R.check_out(bad, ref, bound, name)


# ------------------------------------------------------------------------------------------------ split stem
@pytest.mark.parametrize("dt", [F16, BF16])
def test_split_residue_bounds(dt):
    """The kernel's hi / lo split (fp32 subtraction, then RN to 16 bits): the residue, lo and hi + lo bounds the split
    bound is made of, including fp16 remainders below the smallest normal (2^-14)."""
    g = torch.Generator().manual_seed(3)
    v = torch.cat([torch.rand(20000, generator=g), torch.randn(20000, generator=g) * 0.2,
                   torch.rand(20000, generator=g) * 2.0 ** -8, torch.rand(2000, generator=g) * 2.0 ** -20])
    hi, lo = D.split16(v, dt)
    u, eta = _U16[dt], _ETA[dt]
    va = v.double().abs()
    r = (v.double() - hi.double() - lo.double()).abs()
    assert bool((r <= u * u * va + eta).all())
    assert bool((lo.double().abs() <= (u + u * u) * va + 2 * eta).all())
    assert bool((hi.double().abs() + lo.double().abs() <= (1 + u) ** 2 * va + 3 * eta).all())
    if dt == F16:
        sub = lo.abs() < 2.0 ** -14
        assert int((sub & (lo != 0)).sum()) > 1000, "the case has no subnormal fp16 remainders"
        assert float(r[sub].max()) > 0, "no remainder was rounded in the subnormal range"
        assert bool((r > u * u * va).any()), "the eta term is needed: some residue exceeds u^2 |v|"


@pytest.mark.parametrize("dt", [F16, BF16])
def test_split_stem_bound_holds_and_has_teeth(dt):
    """A float32 emulation of the split stem (K = 96, products of 16-bit hi / lo parts, fp32 accumulation, epilogue,
    16-bit store) lies within stem_split_bound of the float64 conv of the unrounded operands; known-wrong outputs do
    not.  And the batch sums in the kernel's order lie within sums_bound, a missing tile does not."""
    n, h, w = 2, 6, 10
    x, wt, sc, sh = _case(7, n, h, w)
    xh, xl = D.split16(x, dt)
    wh, wl = D.split16(wt, dt)

    def cols(t, drop):
        c = R.im2col(t.double(), 3, 1, 1).numpy()
        return _drop_border_tap(c, w, 3) if drop else c
    wmat = lambda t: t.reshape(32, -1).t().double().numpy()               # noqa: E731
    b = np.concatenate([wmat(wh), wmat(wh), wmat(wl)], 0)

    def emulate(drop, shift):
        a = np.concatenate([cols(xh, drop), cols(xl, drop), cols(xh, drop)], 1)
        return _store(_epi(_mma_acc(a, b), sc.numpy(), shift.numpy(), True), dt)
    got = emulate(False, sh)
    raw, S = R.conv_raw(x, wt, 1, 1)
    ref = R.epilogue(raw, sc, sh, leaky=True)
    Aw = wt.double().abs().reshape(32, -1).sum(1)
    bound = D.stem_split_bound(ref, S, D.stem_patch_abs(x), Aw, dt, scale=sc, shift=sh)
    _assert_teeth(got, ref, bound, _faults(emulate, got, sh, n, h, w))
    # the batch sums: each (CTA, warp, lane) chain adds 32 pixels of every tile of its CTA, then one atomic per chain
    z = got.float().numpy()                                              # stored values, exact in fp32
    zi = z.reshape(n, h, w, 32)
    th, tw = -(-h // 8), -(-w // 16)
    tiles = n * th * tw
    grid = min(tiles, 8 * SMS)
    s0 = np.full(32, 3.0, np.float32)
    total = s0.copy()
    for cta in range(grid):
        for warp in range(4):
            chain = np.zeros(32, np.float32)
            for t in range(cta, tiles, grid):
                img, ty, tx = t // (th * tw), (t // tw) % th, t % tw
                for px in range(32 * warp, 32 * warp + 32):
                    y, xx = ty * 8 + px // 16, tx * 16 + px % 16
                    if y < h and xx < w:
                        chain = _f32(chain + zi[img, y, xx])
            total = _f32(total + chain)
    depth = D.sums_depth(tiles, SMS)
    zt = torch.from_numpy(z).double()
    b_s, _ = D.sums_bound(zt, torch.from_numpy(s0), torch.zeros(32), depth)
    want = torch.from_numpy(s0).double() + zt.sum(0)
    R.check_out(torch.from_numpy(total), want, b_s, "sums")
    with pytest.raises(AssertionError):                                   # one tile missing from the sums
        R.check_out(torch.from_numpy(total) - zt.reshape(n, h, w, 32)[1, :8, :16].sum((0, 1)), want, b_s, "tile missing")


def test_split_bound_is_tight_enough_for_bf16():
    """On bf16 operands rounded once (no split) the stem misses its float64 value by more than the split bound
    allows: the split bound checks that the lo parts are used."""
    dt = BF16
    x, wt, sc, sh = _case(9)
    raw, S = R.conv_raw(x, wt, 1, 1)
    plain, _ = R.conv_raw(x.to(dt), wt.to(dt), 1, 1)
    Aw = wt.double().abs().reshape(32, -1).sum(1)
    e = D.split_bound(S, D.stem_patch_abs(x), Aw, dt) + R.C_STEP * D.SPLIT_N16 * D.split_mag(S, D.stem_patch_abs(x), Aw, dt)
    assert bool(((plain - raw).abs() > e).any())


# ------------------------------------------------------------------------------------------------ other stems, halo / thin
@pytest.mark.parametrize("dt", [F16, BF16])
def test_cuda_stem_bound_holds_and_has_teeth(dt):
    """The CUDA-core stem: a 27-term float32 fmaf chain in (r, s, ci) order on the unrounded operands."""
    n, h, w = 2, 6, 10
    x, wt, sc, sh = _case(11, n, h, w)
    wm = wt.reshape(32, -1).t().double().numpy()

    def emulate(drop, shift):
        cols = R.im2col(x.double(), 3, 1, 1).numpy()
        if drop:
            cols = _drop_border_tap(cols, w, 3)
        acc = np.zeros((cols.shape[0], 32), np.float32)
        for k in range(27):
            acc = _fma(np.broadcast_to(_f32(cols[:, k:k + 1]), acc.shape), np.broadcast_to(_f32(wm[k]), acc.shape), acc)
        return _store(_epi(acc, sc.numpy(), shift.numpy(), True), dt)
    got = emulate(False, sh)
    raw, S = R.conv_raw(x, wt, 1, 1)
    ref = R.epilogue(raw, sc, sh, leaky=True)
    bound = D.cuda_stem_bound(ref, S, dt, scale=sc, shift=sh)
    _assert_teeth(got, ref, bound, _faults(emulate, got, sh, n, h, w))


@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("kind", ["stem", "thin"])
def test_mma_bounds_hold_and_have_teeth(dt, kind):
    """The plain mma.sync stem (n16 = 2, K = 27 padded to 32) and the thin kernel (n16 = 18) on RN16 operands, with the
    thin kernel's residual: fp32 accumulation in k order, epilogue, store."""
    n, h, w = 2, 6, 10
    cin, cout, n16 = (3, 32, D.STEM_N16) if kind == "stem" else (32, 64, D.THIN_N16)
    x, wt, sc, sh = _case(13, n, h, w, cin, cout)
    x16, w16 = x.to(dt), wt.to(dt)
    res = torch.randn((n * h * w, cout), generator=torch.Generator().manual_seed(1)).to(dt) if kind == "thin" else None
    wm = w16.reshape(cout, -1).t().double().numpy()

    def emulate(drop, shift):
        cols = R.im2col(x16.double(), 3, 1, 1).numpy()
        if drop:
            cols = _drop_border_tap(cols, w, cin)
        v = _epi(_mma_acc(cols, wm), sc.numpy(), shift.numpy(), True)
        if res is not None:
            v = _f32(v + res.float().numpy())
        return _store(v, dt)
    got = emulate(False, sh)
    raw, S = R.conv_raw(x16, w16, 1, 1)
    ref = R.epilogue(raw, sc, sh, leaky=True, res=res)
    bound = R.out_bound(ref, S, n16, dt, scale=sc, shift=sh, res=res)
    _assert_teeth(got, ref, bound, _faults(emulate, got, sh, n, h, w))


@pytest.mark.parametrize("dt", [F16, BF16])
def test_fused_interval_contains_the_stored_stem(dt):
    """Any stem value within e0 of the float64 value rounds into [x* - d, x* + d], and Conv_1 on such values lies within
    the interval bound."""
    n, h, w = 1, 8, 16
    x, w0, s0, b0 = _case(17, n, h, w)
    g = torch.Generator().manual_seed(2)
    w1 = (torch.randn((64, 3, 3, 32), generator=g) / (3 * 32 ** 0.5)).to(dt)
    s1, b1 = torch.rand(64, generator=g) + 0.5, torch.randn(64, generator=g) * 0.1
    raw0, S0 = R.conv_raw(x.to(dt), w0.to(dt), 1, 1)
    v0 = R.epilogue(raw0, s0, b0, leaky=True)
    e0 = R.out_bound(v0, S0, D.STEM_N16, torch.float32, scale=s0, shift=b0)
    xs, d = D.stem_interval(v0, S0, dt, s0, b0)
    for t in (-1.0, -0.5, 0.0, 0.5, 1.0):
        stored = D.rn16(v0 + t * e0, dt)
        assert bool(((stored - xs).abs() <= d).all())
    stored = D.rn16(v0 - e0, dt).reshape(1, h, w, 32)
    raw, S, extra = D.conv1_on_interval(xs.reshape(1, h, w, 32), d.reshape(1, h, w, 32), w1, 2, s1)
    ref = R.epilogue(raw, s1, b1, leaky=True)
    e32 = R.out_bound(ref, S, 18, torch.float32, scale=s1, shift=b1) + extra
    bound = e32 + 0.5 * R.ulp(ref.abs() + e32, dt)
    r1, _ = R.conv_raw(stored, w1, 2, 1)
    got = D.rn16(R.epilogue(r1, s1, b1, leaky=True), dt)
    R.check_out(got, ref, bound, "Conv_1 on the low end of the interval")
    assert float(d.max()) > 0, "the case has no stem value near a rounding midpoint"
