"""The direct forward conv kernels against float64 (tests/direct_ref.py): the halo-tile conv and the fused stem + Conv_1
(csrc/conv_halo.cu), the mma.sync thin kernel and stems (csrc/conv_thin.cu) and the CUDA-core stem (csrc/layers.cu).

One case table (HALO_CASES, THIN_CASES, STEM_CASES, FUSED_CASES) covers every instantiation of halo_kernel_type and
thin_kernel_type in both 16-bit types (tests/test_conv_direct_host.py asserts that).  Each halo instantiation has a
small case (partial bottom tile with an odd output height, n >= 3 so that tiles cross images, channel slices of wider
input, output and residual buffers) and a deep case with at least 17 tiles per CTA, which wraps every operand ring
(at most 6 halo stages, 8 image stages for the fused stem) at least twice.

Every case runs
  - on float operands, within the per-element float64 bound (worst err / bound printed on a "DIRECT" line);
  - where its entry point can turn leaky off, once more on small-integer operands (image k / 8 for the stems), where
    every product, partial sum and stored value is exact: the output (and the stem's batch sums) must equal the float64
    reference bit for bit, so a wrong tap, pixel, row or channel fails however small its contribution.
Buffer hygiene: the output sits between guard rows, and everything outside its channel slice is filled with 0xFF
bytes (NaN in both 16-bit types), as are the input's and residual's unused channels: no byte outside the output slice
may change, the inputs must be unchanged, and two launches must give identical bits."""
import ctypes as C
import time
import zlib

import pytest
import torch

from tests import conv_ref as R
from tests import direct_ref as D

pytestmark = pytest.mark.gpu
F16, BF16 = torch.float16, torch.bfloat16
GUARD = 3                          # guard rows of out_ld elements before and after every output
DEEP_TILES = 17                    # tiles per CTA of a deep halo case: every ring (<= 8 stages) wraps twice
OPTS = ("YB_CONV_RES", "YB_STEM_SPLIT")
U32_PRODUCT = R.U32                # the e4m3 output's value x (1 / s_out) product rounds once in fp32


@pytest.fixture
def L():
    from yolov3_tensorflow_b200 import _lib
    for k in OPTS:
        _lib.set_option(k, None)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield _lib
    for k in OPTS:
        _lib.set_option(k, None)
    print(f"DIRECT time {time.time() - t0:.1f} s, peak CUDA memory {torch.cuda.max_memory_allocated() / 2 ** 20:.0f} MiB")


def _sms(L):
    s = C.c_int()
    L.check(L.lib.yb_device_info(C.byref(s), None, None), "device_info")
    return s.value


def _seed(name):
    return zlib.crc32(name.encode()) % 1000 * 2


def _code(L, dt):
    return L.YB_F16 if dt == F16 else L.YB_BF16


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g, device="cuda").float()


# ------------------------------------------------------------------------------------------------------ case table
def halo_key(dt, cin, cout, s, res=False, ldg=False, stem=False, e4m3=False):
    """The conv_halo_kernel instantiation a launch selects (halo_select): (dtype, cin, cout, stride, fused stem, e4m3
    output, residual box)."""
    box = res and not ldg and not stem and (cin, cout, s) == (32, 64, 1)
    return (dt, cin, cout, s, stem, e4m3, box)


def thin_key(dt, cout, s, stem=False, split=False):
    return (dt, cout, s, stem, split)


class Case:
    def __init__(self, name, n, h, w, cin, cout, s, dt, res=False, ldg=False, deep=False, extra=True):
        self.name, self.n, self.h, self.w, self.cin, self.cout, self.s, self.dt = name, n, h, w, cin, cout, s, dt
        self.res, self.ldg, self.deep = res, ldg, deep
        # channel slices: input at offset 16 of cin + 32, output at 8 of cout + 16, residual at 8 of cout + 8
        self.in_off, self.in_ld = (16, cin + 32) if extra else (0, cin)
        self.out_off, self.out_ld = (8, cout + 16) if extra else (0, cout)
        self.res_off, self.res_ld = (8, cout + 8) if extra else (0, cout)

    def __repr__(self):
        return self.name


def _halo_cases():
    cases = []
    # (cin, cout, stride): small (n, h, w), deep (n, h, w) on real layer geometries
    geo = {(32, 64, 1): ((3, 21, 24), (7, 208, 208)),     # Conv_3 at 416
           (32, 64, 2): ((3, 42, 48), (7, 416, 416)),     # Conv_1 at 416
           (32, 128, 1): ((3, 21, 24), (7, 208, 208)),
           (32, 128, 2): ((3, 42, 48), (7, 416, 416)),
           (64, 64, 1): ((3, 21, 24), (25, 104, 104)),
           (64, 64, 2): ((3, 42, 48), (25, 208, 208)),
           (64, 128, 1): ((3, 21, 24), (25, 104, 104))}   # Conv_6 / Conv_8 at 416
    for dt in (F16, BF16):
        t = "f16" if dt == F16 else "bf16"
        for (ci, co, s), (small, deep) in geo.items():
            variants = [(False, False)]
            if (ci, co, s) == (32, 64, 1):
                variants += [(True, False), (True, True)]          # the residual box, and YB_CONV_RES=ldg
            if (ci, co, s) == (64, 128, 1):
                variants += [(True, False)]                         # global-read residual, staging epilogue
            for res, ldg in variants:
                tag = f"halo-{ci}-{co}-s{s}-{t}" + ("-res" if res else "") + ("-ldg" if ldg else "")
                cases.append(Case(tag + "-small", *small, ci, co, s, dt, res, ldg))
                cases.append(Case(tag + "-deep", *deep, ci, co, s, dt, res, ldg, deep=True))
    # the shapes of the earlier halo test
    for i, (n, h, w, ci, co, s, res, dt) in enumerate([
            (2, 32, 16, 64, 128, 1, False, F16), (2, 32, 16, 32, 64, 1, True, F16), (3, 40, 24, 64, 128, 1, True, F16),
            (2, 104, 104, 64, 128, 1, True, BF16), (1, 208, 208, 32, 64, 1, True, F16), (2, 64, 32, 32, 64, 2, False, F16),
            (3, 80, 48, 32, 64, 2, False, BF16), (2, 64, 32, 64, 64, 2, False, F16), (1, 416, 416, 32, 64, 2, False, F16),
            (2, 48, 40, 32, 128, 1, False, F16), (2, 32, 16, 64, 64, 1, True, BF16)]):
        cases.append(Case(f"halo-old{i}-{n}x{h}x{w}-{ci}-{co}-s{s}", n, h, w, ci, co, s, dt, res, extra=bool(i % 2)))
    return cases


def _thin_cases():
    cases = []
    for dt in (F16, BF16):
        t = "f16" if dt == F16 else "bf16"
        for co in (32, 64):
            for s in (1, 2):
                for res in (False, True):
                    # 21 x 37 outputs: partial 8 x 16 tiles in both directions
                    cases.append(Case(f"thin-{co}-s{s}-{t}" + ("-res" if res else ""), 3, 21 * s, 37 * s, 32, co, s, dt, res))
    cases.append(Case("thin-64-s1-f16-res-deep", 10, 208, 208, 32, 64, 1, F16, True, deep=True))
    cases.append(Case("thin-32-s2-bf16-deep", 10, 416, 416, 32, 32, 2, BF16, deep=True))
    for i, (n, h, w, co, s, res, dt) in enumerate([(2, 32, 48, 64, 1, True, F16), (2, 64, 96, 64, 2, False, F16),
                                                   (1, 40, 24, 64, 1, False, BF16), (3, 26, 26, 32, 2, False, F16)]):
        cases.append(Case(f"thin-old{i}-{n}x{h}x{w}-{co}-s{s}", n, h, w, 32, co, s, dt, res, extra=False))
    return cases


HALO_CASES = _halo_cases()
THIN_CASES = _thin_cases()
# stems: (name, kernel, n, h, w, dtype); kernel "tc" (plain mma.sync), "cuda" (CUDA-core), "split" (with batch sums)
STEM_CASES = [(f"stem-{k}-{sh[0]}x{sh[1]}x{sh[2]}-{'f16' if dt == F16 else 'bf16'}", k, *sh, dt)
              for k in ("tc", "cuda", "split") for dt in (F16, BF16) for sh in ((3, 37, 45), (2, 40, 56))]
STEM_TRAIN_CASES = [(f"stem-split-train-{n}x{hw}-{'f16' if dt == F16 else 'bf16'}", n, hw, dt)
                    for n, hw in ((32, 416), (32, 608)) for dt in (F16, BF16)]
FUSED_CASES = [(2, 64, 32, F16), (3, 80, 48, BF16), (1, 416, 416, F16), (2, 96, 160, F16), (7, 416, 416, F16),
               (7, 416, 416, BF16)]


def case_keys():
    """Every instantiation key the GPU cases launch (tests/test_conv_direct_host.py checks the tables against it)."""
    halo = {halo_key(c.dt, c.cin, c.cout, c.s, c.res, c.ldg) for c in HALO_CASES}
    halo |= {halo_key(dt, 32, 64, 2, stem=True) for _, _, _, dt in FUSED_CASES}
    halo |= {halo_key(F16, 32, 64, 1, True, ldg, e4m3=True) for ldg in (False, True)}     # test_e4m3_conv3
    thin = {thin_key(c.dt, c.cout, c.s) for c in THIN_CASES}
    thin |= {thin_key(c[5], 32, 1, True, c[1] == "split") for c in STEM_CASES if c[1] != "cuda"}
    return halo, thin


# ------------------------------------------------------------------------------------------------------ buffers
class Out:
    """A [n, ho, wo, ld] output with GUARD rows before and after, all 0xFF bytes; the view is channels [off, off + c)."""

    def __init__(self, n, ho, wo, ld, off, c, dt):
        self.rows, self.ld, self.off, self.c = n * ho * wo, ld, off, c
        self.buf = torch.empty(((self.rows + 2 * GUARD) * ld,), dtype=dt, device="cuda")
        self.buf.view(torch.int16).fill_(-1)
        self.view = self.buf[GUARD * ld:(GUARD + self.rows) * ld].view(n, ho, wo, ld)[..., off:off + c]

    def ptr(self):
        return C.c_void_p(self.view.data_ptr())

    def check_outside(self, what):
        b = self.buf.view(torch.int16).view(-1, self.ld)
        mask = torch.ones_like(b, dtype=torch.bool)
        mask[GUARD:GUARD + self.rows, self.off:self.off + self.c] = False
        bad = int((b[mask] != -1).sum())
        assert bad == 0, f"{what}: {bad} elements outside the output slice or in the guard rows were written"


def _slice_of_poison(shape, ld, off, values):
    """values [..., c] placed at channels [off, off + c) of a 0xFF-filled [..., ld] buffer; returns (buffer, view)."""
    buf = torch.empty(shape[:-1] + (ld,), dtype=values.dtype, device="cuda")
    buf.view(torch.int16).fill_(-1)
    view = buf[..., off:off + shape[-1]]
    view.copy_(values)
    return buf, view


def _launch_twice(launch, outs, inputs, what):
    """Runs launch() twice: the second launch must reproduce the first's bits, the inputs must be unchanged."""
    snaps = [_bits(t).clone() for t in inputs]
    launch()
    torch.cuda.synchronize()
    first = [_bits(o.buf).clone() for o in outs]
    launch()
    torch.cuda.synchronize()
    for o, f in zip(outs, first):
        assert torch.equal(_bits(o.buf), f), f"{what}: a second launch gave different bits"
        o.check_outside(what)
    for t, s in zip(inputs, snaps):
        assert torch.equal(_bits(t), s), f"{what}: an input buffer changed"


def _check(got, ref, bound, exact, what):
    """Exact operands: bit for bit (premise: the reference is representable); float: within the bound."""
    if exact:
        dt = got.dtype
        assert torch.equal(D.rn16(ref, dt), ref), f"{what}: premise: the exact reference is not representable in {dt}"
        bad = int((got.double() != ref).sum())
        assert bad == 0, f"{what}: {bad} elements differ from the exact reference"
        return 0.0
    return R.check_out(got, ref, bound, what)


def _report(name, exact, frac, extra=""):
    print(f"DIRECT {name} {'exact' if exact else 'float'}: " +
          ("bit-identical to float64" if exact else f"worst err/bound {frac:.3f}") + extra)


# ------------------------------------------------------------------------------------------------------ halo / thin
def _layer_operands(c, exact, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ho, wo = c.h // c.s, c.w // c.s
    if exact:
        x = _ints((c.n, c.h, c.w, c.cin), -1, 1, g)
        wt = _ints((c.cout, 3, 3, c.cin), -1, 1, g)
        sc, sh = _ints((c.cout,), 1, 2, g), _ints((c.cout,), -2, 2, g)
        r = _ints((c.n, ho, wo, c.cout), -4, 4, g)
    else:
        x = torch.randn((c.n, c.h, c.w, c.cin), generator=g, device="cuda")
        wt = torch.randn((c.cout, 3, 3, c.cin), generator=g, device="cuda") / (3 * c.cin ** 0.5)
        sc = torch.rand((c.cout,), generator=g, device="cuda") + 0.5
        sh = torch.randn((c.cout,), generator=g, device="cuda") * 0.1
        r = torch.randn((c.n, ho, wo, c.cout), generator=g, device="cuda")
    return x.to(c.dt), wt, sc, sh, r.to(c.dt)


def _run_layer(L, c, kind, exact):
    dt, code = c.dt, _code(L, c.dt)
    ho, wo = c.h // c.s, c.w // c.s
    x, wt, sc, sh, r = _layer_operands(c, exact, seed=_seed(c.name) + exact)
    cp = L.lib.yb_conv_cout_pad(c.cout)
    wp = torch.zeros((cp, 3, 3, c.cin), dtype=dt, device="cuda")
    L.check(L.lib.yb_pack_conv_weights(L.ptr(wt), L.YB_W_OHWI, c.cout, c.cin, 3, cp, code, L.ptr(wp), L.stream_handle()), "pack")
    scp = torch.ones(cp, device="cuda"); scp[:c.cout] = sc
    shp = torch.zeros(cp, device="cuda"); shp[:c.cout] = sh
    xbuf, xv = _slice_of_poison(x.shape, c.in_ld, c.in_off, x)
    rbuf, rv = _slice_of_poison(r.shape, c.res_ld, c.res_off, r) if c.res else (None, None)
    out = Out(c.n, ho, wo, c.out_ld, c.out_off, c.cout, dt)
    leaky = 0 if exact else 1
    d = L.ConvDesc(n=c.n, h=c.h, w=c.w, cin=c.cin, cout=c.cout, ksize=3, stride=c.s, in_ld=c.in_ld, out_ld=c.out_ld,
                   res_ld=c.res_ld, dtype=code, out_fp32=0, leaky=leaky, upsample2x=0)
    fn = L.lib.yb_conv3x3_halo_fwd if kind == "halo" else L.lib.yb_conv3x3_thin_fwd
    if kind == "halo":
        assert L.lib.yb_conv3x3_halo_supported(C.byref(d)) == 1
    L.set_option("YB_CONV_RES", "ldg" if c.ldg else None)

    def launch():
        L.check(fn(C.byref(d), C.c_void_p(xv.data_ptr()), L.ptr(wp), L.ptr(scp), L.ptr(shp),
                   None if rv is None else C.c_void_p(rv.data_ptr()), out.ptr(), L.stream_handle()), kind)
    _launch_twice(launch, [out], [xbuf, wp] + ([rbuf] if c.res else []), c.name)
    L.set_option("YB_CONV_RES", None)
    n16 = D.halo_n16(c.cin) if kind == "halo" else D.THIN_N16
    worst = 0.0
    for i in range(c.n):
        raw, S = R.conv_raw(xv[i:i + 1], wp[:c.cout], c.s, 1)
        res = rv[i].reshape(-1, c.cout) if c.res else None
        ref = R.epilogue(raw, sc, sh, leaky=bool(leaky), res=res)
        bound = R.out_bound(ref, S, n16, dt, scale=sc, shift=sh, res=res)
        worst = max(worst, _check(out.view[i].reshape(-1, c.cout), ref, bound, exact, f"{c.name} image {i}"))
        del raw, S, ref, bound
    _report(c.name, exact, worst)


def _deep_premise(L, name, tiles, max_grid):
    sms = _sms(L)
    grid = min(tiles, max_grid(sms))
    per_cta = -(-tiles // grid)
    print(f"DIRECT {name} premise: {tiles} tiles on a grid of at most {grid} CTAs ({sms} SMs): {per_cta} tiles per CTA")
    return per_cta


@pytest.mark.parametrize("c", HALO_CASES, ids=[c.name for c in HALO_CASES])
def test_halo_conv(L, c):
    if c.deep:
        tiles = c.n * -(-(c.h // c.s) // 16) * (c.w // c.s // 8)
        assert _deep_premise(L, c.name, tiles, lambda sms: sms) >= DEEP_TILES
    for exact in (False, True):
        _run_layer(L, c, "halo", exact)


@pytest.mark.parametrize("c", THIN_CASES, ids=[c.name for c in THIN_CASES])
def test_thin_conv(L, c):
    if c.deep:
        tiles = c.n * -(-(c.h // c.s) // 8) * -(-(c.w // c.s) // 16)
        assert tiles >= 3 * 8 * _sms(L), "fewer than 3 tiles per CTA at SMs x 8 CTAs"
        _deep_premise(L, c.name, tiles, lambda sms: 8 * sms)
    for exact in (False, True):
        _run_layer(L, c, "thin", exact)


# ------------------------------------------------------------------------------------------------------ stems
def _stem_operands(n, h, w, exact, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if exact:       # image k / 8, integer weights, scale and shift: |value| <= 27 * 0.5 * 2 + 2 < 32, multiples of 1/8
        x = _ints((n, h, w, 3), -4, 4, g) / 8
        wt = _ints((32, 3, 3, 3), -1, 1, g)
        return x, wt, _ints((32,), 1, 2, g), _ints((32,), -2, 2, g)
    x = torch.rand((n, h, w, 3), generator=g, device="cuda")
    wt = torch.randn((32, 3, 3, 3), generator=g, device="cuda") * 0.2
    return x, wt, torch.rand((32,), generator=g, device="cuda") + 0.5, torch.randn((32,), generator=g, device="cuda") * 0.1


def _stem_launch(L, kind, x, wt, sc, sh, n, h, w, dt, leaky, out, sums=None):
    code, st = _code(L, dt), L.stream_handle()
    if kind == "cuda":
        L.check(L.lib.yb_stem_conv_fwd(L.ptr(x), L.ptr(wt), L.ptr(sc), L.ptr(sh), n, h, w, 32, code, leaky, out.ptr(), st), "stem")
    elif sums is None:
        L.check(L.lib.yb_stem_conv_fwd_tc(L.ptr(x), L.ptr(wt), L.ptr(sc), L.ptr(sh), n, h, w, code, leaky, out.ptr(), st), "stem_tc")
    else:
        L.check(L.lib.yb_stem_conv_fwd_tc_stats(L.ptr(x), L.ptr(wt), L.ptr(sc), L.ptr(sh), n, h, w, code, leaky, out.ptr(),
                                                L.ptr(sums[0]), L.ptr(sums[1]), st), "stem_tc_stats")


def _stem_ref(kind, x, wt, sc, sh, leaky, dt):
    """(ref, bound) [h w, 32] of one image x [1, h, w, 3] (float32) for stem kernel `kind`."""
    if kind == "tc":
        raw, S = R.conv_raw(x.to(dt), wt.to(dt), 1, 1)
        ref = R.epilogue(raw, sc, sh, leaky=leaky)
        return ref, R.out_bound(ref, S, D.STEM_N16, dt, scale=sc, shift=sh)
    raw, S = R.conv_raw(x, wt, 1, 1)
    ref = R.epilogue(raw, sc, sh, leaky=leaky)
    if kind == "cuda":
        return ref, D.cuda_stem_bound(ref, S, dt, scale=sc, shift=sh)
    Aw = wt.double().abs().reshape(32, -1).sum(1)
    return ref, D.stem_split_bound(ref, S, D.stem_patch_abs(x), Aw, dt, scale=sc, shift=sh)


def _run_stem(L, name, kind, n, h, w, dt, exact, scale_one=False):
    x, wt, sc, sh = _stem_operands(n, h, w, exact, seed=_seed(name) + exact)
    if scale_one:                  # the training forward's: scale 1, shift 0, leaky off
        sc, sh = torch.ones_like(sc), torch.zeros_like(sh)
    leaky = 0 if exact or scale_one else 1
    out = Out(n, h, w, 32, 0, 32, dt)
    sums = None
    if kind == "split":
        g = torch.Generator(device="cuda").manual_seed(5)
        s0, q0 = _ints((32,), -64, 64, g), _ints((32,), 0, 64, g)        # the kernel accumulates onto these
        sums = (torch.empty_like(s0), torch.empty_like(q0))

    def launch():
        if sums is not None:
            sums[0].copy_(s0)
            sums[1].copy_(q0)
        _stem_launch(L, kind, x, wt, sc, sh, n, h, w, dt, leaky, out, sums)
    _launch_twice(launch, [out], [x, wt], name)
    got_sums = None if sums is None else (sums[0].clone(), sums[1].clone())
    worst = 0.0
    zs, zq = torch.zeros(32, dtype=torch.float64, device="cuda"), torch.zeros(32, dtype=torch.float64, device="cuda")
    zabs, zsq = torch.zeros_like(zs), torch.zeros_like(zs)
    for i in range(n):
        ref, bound = _stem_ref(kind, x[i:i + 1], wt, sc, sh, bool(leaky), dt)
        z = out.view[i].reshape(-1, 32)
        worst = max(worst, _check(z, ref, bound, exact, f"{name} image {i}"))
        zd = z.double()
        zs += zd.sum(0); zq += (zd * zd).sum(0)
        zabs += zd.abs().sum(0)
        del ref, bound
    extra = ""
    if got_sums is not None:
        tiles = n * -(-h // 8) * -(-w // 16)
        depth = D.sums_depth(tiles, _sms(L))
        ref_s, ref_q = s0.double() + zs, q0.double() + zq
        b_s = depth * D.U32 * (s0.double().abs() + zabs)
        b_q = depth * D.U32 * (q0.double().abs() + zq)
        if exact:
            # premise: every partial sum is a multiple of 1/8 (1/64 for z^2) below 2^24 of those units
            assert float((s0.abs().double() + zabs).max()) * 8 < 2 ** 24 and float((q0.double() + zq).max()) * 64 < 2 ** 24
            assert torch.equal(got_sums[0].double(), ref_s), f"{name}: batch sums differ from the exact reference"
            assert torch.equal(got_sums[1].double(), ref_q), f"{name}: batch sums of squares differ from the exact reference"
        else:
            fs = R.check_out(got_sums[0], ref_s, b_s, f"{name} sum z")
            fq = R.check_out(got_sums[1], ref_q, b_q, f"{name} sum z^2")
            extra = f", sums {fs:.3f} / {fq:.3f} (depth {depth})"
    _report(name, exact, worst, extra)
    return out


@pytest.mark.parametrize("name,kind,n,h,w,dt", STEM_CASES, ids=[c[0] for c in STEM_CASES])
def test_stem(L, name, kind, n, h, w, dt):
    for exact in (False, True):
        out = _run_stem(L, name, kind, n, h, w, dt, exact)
    if kind == "split":
        # YB_STEM_SPLIT=0: the statistics form multiplies plain 16-bit operands and gives the plain kernel's bits.  On
        # float operands the split form's bits differ from the plain kernel's, so this comparison can fail.
        x, wt, sc, sh = _stem_operands(n, h, w, False, seed=_seed(name) + 1)
        outs = {}
        for mode in ("plain", "nosplit", "split"):
            outs[mode] = Out(n, h, w, 32, 0, 32, dt)
            L.set_option("YB_STEM_SPLIT", "0" if mode == "nosplit" else None)
            sums = None if mode == "plain" else (torch.zeros(32, device="cuda"), torch.zeros(32, device="cuda"))
            _stem_launch(L, "tc" if mode == "plain" else "split", x, wt, sc, sh, n, h, w, dt, 1, outs[mode], sums)
        L.set_option("YB_STEM_SPLIT", None)
        torch.cuda.synchronize()
        plain, nosplit, split = (_bits(outs[k].buf) for k in ("plain", "nosplit", "split"))
        assert torch.equal(plain, nosplit), "YB_STEM_SPLIT=0 differs from the plain kernel"
        differ = int((split != plain).sum())
        assert differ > 0, "premise: on float operands the split kernel gives the plain kernel's bits"
        # exact operands: every lo part is zero, so the split kernel's output is the plain kernel's
        x, wt, sc, sh = _stem_operands(n, h, w, True, seed=_seed(name) + 1)
        plain_exact = Out(n, h, w, 32, 0, 32, dt)
        _stem_launch(L, "tc", x, wt, sc, sh, n, h, w, dt, 0, plain_exact)
        torch.cuda.synchronize()
        assert torch.equal(_bits(out.buf), _bits(plain_exact.buf)), "exact operands: the split kernel differs from the plain one"
        print(f"DIRECT {name}: YB_STEM_SPLIT=0 gives the plain kernel's bits; the split form differs from them in "
              f"{differ} of {plain.numel()} elements")


@pytest.mark.parametrize("name,n,hw,dt", STEM_TRAIN_CASES, ids=[c[0] for c in STEM_TRAIN_CASES])
def test_stem_split_training_shapes(L, name, n, hw, dt):
    """The split stem with its batch sums at the benchmark's training shapes, as the training step calls it."""
    _run_stem(L, name, "split", n, hw, hw, dt, False, scale_one=True)


# ------------------------------------------------------------------------------------------------------ fused stem + Conv_1
@pytest.mark.parametrize("n,h,w,dt", FUSED_CASES)
def test_stem_conv1_fused(L, n, h, w, dt):
    """yb_stem_conv1_fused_fwd within the interval bound (tests/direct_ref.py), and the two-launch path (plain stem,
    then Conv_1 on its stored output) each launch within its own bound."""
    name = f"fused-{n}x{h}x{w}-{'f16' if dt == F16 else 'bf16'}"
    code, st = _code(L, dt), L.stream_handle()
    tiles = n * -(-(h // 2) // 16) * (w // 2 // 8)
    deep = _deep_premise(L, name, tiles, lambda sms: sms)
    if n >= 7:
        assert deep >= DEEP_TILES
    g = torch.Generator(device="cuda").manual_seed(5 + h)
    x = torch.rand((n, h, w, 3), generator=g, device="cuda")
    w0 = torch.randn((32, 3, 3, 3), generator=g, device="cuda") / 5.0
    s0, b0 = torch.rand(32, generator=g, device="cuda") + 0.5, torch.randn(32, generator=g, device="cuda") * 0.1
    w1 = torch.randn((64, 3, 3, 32), generator=g, device="cuda") / (3 * 32 ** 0.5)
    s1, b1 = torch.rand(64, generator=g, device="cuda") + 0.5, torch.randn(64, generator=g, device="cuda") * 0.1
    w1p = torch.zeros((64, 3, 3, 32), dtype=dt, device="cuda")
    L.check(L.lib.yb_pack_conv_weights(L.ptr(w1), L.YB_W_OHWI, 64, 32, 3, 64, code, L.ptr(w1p), st), "pack")
    ho, wo = h // 2, w // 2
    a0 = Out(n, h, w, 32, 0, 32, dt)
    two = Out(n, ho, wo, 64, 0, 64, dt)
    one = Out(n, ho, wo, 80, 8, 64, dt)
    d = L.ConvDesc(n=n, h=h, w=w, cin=32, cout=64, ksize=3, stride=2, in_ld=32, out_ld=64, res_ld=0, dtype=code,
                   out_fp32=0, leaky=1, upsample2x=0)
    d1 = L.ConvDesc(n=n, h=h, w=w, cin=32, cout=64, ksize=3, stride=2, in_ld=32, out_ld=80, res_ld=0, dtype=code,
                    out_fp32=0, leaky=1, upsample2x=0)

    def launch_two():
        L.check(L.lib.yb_stem_conv_fwd_tc(L.ptr(x), L.ptr(w0), L.ptr(s0), L.ptr(b0), n, h, w, code, 1, a0.ptr(), st), "stem")
        L.check(L.lib.yb_conv2d_fwd(C.byref(d), a0.ptr(), L.ptr(w1p), L.ptr(s1), L.ptr(b1), None, two.ptr(), None, None, st),
                "conv1")

    def launch_one():
        L.check(L.lib.yb_stem_conv1_fused_fwd(C.byref(d1), L.ptr(x), L.ptr(w0), L.ptr(s0), L.ptr(b0), L.ptr(w1p), L.ptr(s1),
                                              L.ptr(b1), one.ptr(), st), "fused")
    _launch_twice(launch_two, [a0, two], [x, w0, w1p], name + " two launches")
    _launch_twice(launch_one, [one], [x, w0, w1p], name + " fused")
    w_stem = w0.to(dt)
    worst = {"fused": 0.0, "stem": 0.0, "conv1": 0.0}
    near = 0.0
    for i in range(n):
        raw0, S0 = R.conv_raw(x[i:i + 1].to(dt), w_stem, 1, 1)
        v0 = R.epilogue(raw0, s0, b0, leaky=True)
        b = R.out_bound(v0, S0, D.STEM_N16, dt, scale=s0, shift=b0)
        worst["stem"] = max(worst["stem"], R.check_out(a0.view[i].reshape(-1, 32), v0, b, f"{name} stem image {i}"))
        xs, dd = D.stem_interval(v0, S0, dt, s0, b0)
        near = max(near, float((dd > 0).double().mean()))
        del raw0, S0, b
        raw, S, extra = D.conv1_on_interval(xs.reshape(1, h, w, 32), dd.reshape(1, h, w, 32), w1p, 2, s1)
        ref = R.epilogue(raw, s1, b1, leaky=True)
        e32 = R.out_bound(ref, S, 18, torch.float32, scale=s1, shift=b1) + extra
        bound = e32 + 0.5 * R.ulp(ref.abs() + e32, dt)
        worst["fused"] = max(worst["fused"], R.check_out(one.view[i].reshape(-1, 64), ref, bound, f"{name} fused image {i}"))
        raw, S = R.conv_raw(a0.view[i:i + 1], w1p, 2, 1)
        ref = R.epilogue(raw, s1, b1, leaky=True)
        bound = R.out_bound(ref, S, 18, dt, scale=s1, shift=b1)
        worst["conv1"] = max(worst["conv1"], R.check_out(two.view[i].reshape(-1, 64), ref, bound, f"{name} Conv_1 image {i}"))
        del raw, S, ref, bound, xs, dd
    for k, v in worst.items():
        _report(f"{name} {k}", False, v)
    print(f"DIRECT {name}: at most {near:.2e} of an image's stem values have two candidates")
    _run_two_launch_exact(L, name, n, h, w, dt)


def _run_two_launch_exact(L, name, n, h, w, dt):
    """The two-launch form (the fused kernel always applies leaky to the stem) on exact operands, leaky off: image
    k / 8 with k in {-1, 0, 1}, integer stem weights and scale, Conv_1 weights in {-1, 0, 1} with 1 in 8 nonzero, so
    that every stem value and Conv_1 output is a multiple of 1/8 small enough for both 16-bit types: the stem output
    and Conv_1's output must equal float64 bit for bit."""
    code, st = _code(L, dt), L.stream_handle()
    g = torch.Generator(device="cuda").manual_seed(_seed(name))
    x = _ints((n, h, w, 3), -1, 1, g) / 8
    w0 = _ints((32, 3, 3, 3), -1, 1, g)
    s0, b0 = _ints((32,), 1, 2, g), torch.zeros(32, device="cuda")
    w1 = _ints((64, 3, 3, 32), -1, 1, g) * (_ints((64, 3, 3, 32), 0, 7, g) == 0)
    s1, b1 = torch.ones(64, device="cuda"), _ints((64,), -1, 1, g)
    w1p = torch.zeros((64, 3, 3, 32), dtype=dt, device="cuda")
    L.check(L.lib.yb_pack_conv_weights(L.ptr(w1), L.YB_W_OHWI, 64, 32, 3, 64, code, L.ptr(w1p), st), "pack")
    a0 = Out(n, h, w, 32, 0, 32, dt)
    two = Out(n, h // 2, w // 2, 64, 0, 64, dt)
    d = L.ConvDesc(n=n, h=h, w=w, cin=32, cout=64, ksize=3, stride=2, in_ld=32, out_ld=64, res_ld=0, dtype=code,
                   out_fp32=0, leaky=0, upsample2x=0)

    def launch():
        L.check(L.lib.yb_stem_conv_fwd_tc(L.ptr(x), L.ptr(w0), L.ptr(s0), L.ptr(b0), n, h, w, code, 0, a0.ptr(), st), "stem")
        L.check(L.lib.yb_conv2d_fwd(C.byref(d), a0.ptr(), L.ptr(w1p), L.ptr(s1), L.ptr(b1), None, two.ptr(), None, None, st),
                "conv1")
    _launch_twice(launch, [a0, two], [x, w0, w1p], name + " two launches, exact")
    for i in range(n):
        raw0, _ = R.conv_raw(x[i:i + 1], w0, 1, 1)
        v0 = R.epilogue(raw0, s0, b0)
        _check(a0.view[i].reshape(-1, 32), v0, None, True, f"{name} exact stem image {i}")
        raw1, _ = R.conv_raw(v0.reshape(1, h, w, 32), w1p, 2, 1)
        _check(two.view[i].reshape(-1, 64), R.epilogue(raw1, s1, b1), None, True, f"{name} exact Conv_1 image {i}")
    _report(f"{name} two launches", True, 0.0)


# ------------------------------------------------------------------------------------------------------ e4m3 Conv_3
@pytest.mark.parametrize("ldg", [False, True], ids=["box", "ldg"])
def test_e4m3_conv3(L, ldg):
    """The fp8 plan's Conv_3 (the halo conv's e4m3 output, fp16 in) on the plan's own layer-2 output and layer-1
    residual, at a batch with at least 17 tiles per CTA: the codes against RN(value / s_out) by fp8_ref.check_e4m3, with
    the value's bound conv_ref.out_bound (fp16 operands, n16 = 18) plus the rounding of the 1 / s_out product."""
    import yolov3_tensorflow_b200 as pkg
    from oracle import yolov3_oracle as O
    from tests import fp8_ref as F8
    from tests import infer_plan_ref as P
    from tests.synth import gen_inputs
    n, hw = 7, 416
    L.set_option("YB_CONV_RES", "ldg" if ldg else None)
    m = pkg.yolov3(80, O.COCO_ANCHORS, dtype="fp16")
    m.set_params(O.make_params(80, seed=7, random_bn=True, det_scale=8.0, conf_bias=-2.0), "HWIO")
    x = torch.from_numpy(gen_inputs(29, n, hw, hw)).cuda()
    qm = m.quantize_fp8([x])
    qm.forward(x)
    torch.cuda.synchronize()
    pl = qm._last_plan
    s = P.layer_schedules(L, pl.handle)[3]
    assert s.kernel == L.YB_LAYER_HALO and bool(s.res_smem) == (not ldg), (s.kernel, s.res_smem)
    info = pl.layer_info(3)
    assert (info.cin, info.cout, info.stride) == (32, 64, 1)
    tiles = n * -(-info.out_h // 16) * (info.out_w // 8)
    assert _deep_premise(L, f"e4m3-conv3-{'ldg' if ldg else 'box'}", tiles, lambda sms: sms) >= DEEP_TILES
    p = pl.conv_params(3)
    sc = torch.empty(64, device="cuda")
    sh = torch.empty_like(sc)
    L.check(L.lib.yb_bn_fold(L.ptr(p["gamma"]), L.ptr(p["beta"]), L.ptr(p["mean"]), L.ptr(p["var"]), 64, 1e-5, L.ptr(sc),
                             L.ptr(sh), L.stream_handle()), "bn_fold")
    so = qm.fp8_scales()["act"][3][2]
    inv = float(torch.tensor(1.0, dtype=torch.float32) / torch.tensor(so, dtype=torch.float32))
    w16 = p["w"].half()
    xin, res_t, out = pl.layer_output(2), pl.layer_output(1), pl.layer_output(3)
    assert out.dtype == torch.float8_e4m3fn
    worst = 0.0
    for i in range(n):
        raw, S = R.conv_raw(xin[i:i + 1], w16, 1, 1)
        r = res_t[i].reshape(-1, 64)
        ref = R.epilogue(raw, sc, sh, leaky=True, res=r)
        e32 = R.out_bound(ref, S, 18, torch.float32, scale=sc, shift=sh, res=r)
        bound = e32 + U32_PRODUCT * (ref.abs() + e32)
        got = out[i].reshape(-1, 64).contiguous().view(torch.uint8)
        exact, ulps, near0 = F8.check_e4m3(got, ref * inv, bound * inv, f"e4m3 Conv_3 image {i}")
        worst = max(worst, ulps)
    print(f"DIRECT e4m3-conv3-{'ldg' if ldg else 'box'}: codes equal RN(value / s_out) away from midpoints, worst "
          f"{worst:.2f} e4m3 ulps")
