"""The weight-gradient kernels over deep pipelines, forced split-K and every training layer shape, against float64.

conv_wgrad_kernel (csrc/conv_wgrad.cu) streams its split's 64-pixel blocks through a ring of 4-8 shared-memory stages.
At small shapes the default split-K plan gives every CTA one or two blocks, so the ring never wraps; the training step
runs 6-492 blocks per CTA.  These tests force the split count (YB_WGRAD_SPLITS) so that the blocks per split walk the
ring 0, 1 and 2 times with every residue mod the ring depth, cover the geometries the training plan uses (channel
slices of the concat buffers, cout 32 / 255 / 1024, stride 2 with a dilated dz), and run every distinct wgrad shape of
the 416 x 416 training plan with its own schedule.  Each case asserts its premise through yb_wgrad_schedule, so that a
change of the cost model fails here instead of silently turning a case into a duplicate.

Operands are small integers wherever possible (tests/wgrad_ref.py): then the kernel must equal the float64 reference
bit for bit in every split and atomic order, so a dropped or doubled block, a wrong tap or a stale stage fails at any
size.  Float operands are checked against the float64 bound of wgrad_ref.  Every dw sits between two sentinel rows
holding -0.0, which any stray atomic add changes (-0.0 + 0.0 = +0.0): in training those rows are the neighbouring
layers' gradients.  Each run prints one "WGRAD" line: kernel, blocks per split and their residue mod the ring depth,
split count, grid, and for float operands the worst error as a fraction of the bound."""
import ctypes as C

import pytest
import torch

from tests import conv_ref as R
from tests import wgrad_ref as W

pytestmark = pytest.mark.gpu

KEYS = ("YB_WGRAD_TP", "YB_WGRAD_EPI", "YB_WGRAD_SPLITS", "YB_STEM_WGRAD")
SENT_BITS = -(2 ** 31)            # -0.0f


@pytest.fixture
def L():
    from yolov3_tensorflow_b200 import _lib
    for k in KEYS:
        _lib.set_option(k, None)
    yield _lib
    for k in KEYS:
        _lib.set_option(k, None)


def _code(L, dtype):
    return L.YB_F16 if dtype == torch.float16 else L.YB_BF16


def _sms(L):
    s = C.c_int()
    L.check(L.lib.yb_device_info(C.byref(s), None, None), "device_info")
    return s.value


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g, device="cuda", dtype=torch.int8)


def _poison(shape, g):
    """Nonzero integers: a gather from the wrong place changes the result even where the right place holds zeros."""
    v = _ints(shape, 1, 3, g)
    return torch.where(_ints(shape, 0, 1, g) == 0, v, -v)


class Problem:
    """One yb_conv2d_wgrad problem in the training plan's storage: x a channel slice [in_off, in_off + cin) of an
    [n, h, w, in_ld] buffer, dz [n, ho, wo, dz_ld] (or zero-inserted [n, h, w, dz_ld] when dilated), dw between two
    sentinel rows.  Storage outside the operands holds poison."""

    def __init__(self, L, n, h, w, cin, cout, k, s, dtype=torch.float16, exact=True, in_ld=None, in_off=0,
                 dz_ld=None, dilated=False, seed=0, amp=2):
        self.L, self.dtype, self.exact = L, dtype, exact
        self.k, self.s, self.cout = k, s, cout
        in_ld = in_ld or cin
        dz_ld = dz_ld or cout
        self.dz_ld, self.dilated = dz_ld, dilated
        g = torch.Generator(device="cuda").manual_seed(seed)
        ho, wo = h // s, w // s
        if exact:
            x = _ints((n, h, w, cin), -amp, amp, g).to(dtype)
            dz = _ints((n, ho, wo, cout), -amp, amp, g).to(dtype)
            self.dw0 = _ints((cout, k * k * cin), -64, 64, g).float()
        else:
            x = torch.randn((n, h, w, cin), generator=g, device="cuda").to(dtype)
            dz = (torch.randn((n, ho, wo, cout), generator=g, device="cuda") * 0.1).to(dtype)
            self.dw0 = torch.randn((cout, k * k * cin), generator=g, device="cuda")
        self.xbuf = _poison((n, h, w, in_ld), g).to(dtype)
        self.xbuf[..., in_off:in_off + cin] = x
        self.xp = self.xbuf.data_ptr() + in_off * self.xbuf.element_size()
        if dilated:
            assert s == 2
            self.dzbuf = _poison((n, h, w, dz_ld), g).to(dtype)
            self.dzbuf[:, ::2, ::2, :cout] = dz
            dzc = W.compact_dilated(self.dzbuf)[..., :cout]
        else:
            self.dzbuf = _poison((n, ho, wo, dz_ld), g).to(dtype)
            self.dzbuf[..., :cout] = dz
            dzc = self.dzbuf[..., :cout]
        self.ref, self.S = W.wgrad_ref(x, dzc, k, s)
        self.desc = L.ConvDesc(n=n, h=h, w=w, cin=cin, cout=cout, ksize=k, stride=s, in_ld=in_ld, out_ld=dz_ld, res_ld=0,
                               dtype=_code(L, dtype), out_fp32=0, leaky=0, upsample2x=0)
        self.buf = torch.empty((cout + 2, k * k * cin), dtype=torch.float32, device="cuda")

    def schedule(self):
        info = self.L.WgradSchedule()
        self.L.check(self.L.lib.yb_wgrad_schedule(C.byref(self.desc), _sms(self.L), C.byref(info)), "wgrad_schedule")
        return info

    def run(self, launches=1):
        """Launches on dw0 and returns dw (float32, the sentinel rows checked)."""
        L = self.L
        self.buf.view(torch.int32).fill_(SENT_BITS)
        self.buf[1:-1] = self.dw0
        for _ in range(launches):
            L.check(L.lib.yb_conv2d_wgrad(C.byref(self.desc), C.c_void_p(self.xp), L.ptr(self.dzbuf), self.dz_ld,
                                          int(self.dilated), C.c_void_p(self.buf[1].data_ptr()), L.stream_handle()),
                    "wgrad")
        torch.cuda.synchronize()
        bits = self.buf.view(torch.int32)
        for row, where in ((0, "before"), (-1, "after")):
            bad = int((bits[row] != SENT_BITS).sum())
            assert bad == 0, f"{bad} stray writes into the sentinel row {where} dw"
        return self.buf[1:-1]

    def check(self, name, launches=1):
        """One run against the reference: bit-exact for integer operands, within the float64 bound otherwise."""
        i = self.schedule()
        got = self.run(launches)
        want = self.dw0.double() + launches * self.ref
        line = (f"WGRAD {name}: bnw {i.bnw} tp {i.tp} stages {i.stages} num_kb {i.num_kb} kb/split {i.kb_per_split} "
                f"mod stages {i.kb_per_split % i.stages} splits {i.splits} last {i.num_kb - (i.splits - 1) * i.kb_per_split} "
                f"grid {i.grid_x}x{i.grid_y}x{i.grid_z}")
        if self.exact:
            assert float(launches * self.S.max() + self.dw0.abs().max()) < W.EXACT_LIMIT, f"{name}: operands too large"
            diff = got.double() != want
            if bool(diff.any()):
                idx = tuple(diff.nonzero()[0].tolist())
                raise AssertionError(f"{name}: {int(diff.sum())}/{diff.numel()} elements differ from the exact result; "
                                     f"first at {idx}: got {float(got[idx])} want {float(want[idx])}")
            print(line + " exact")
        else:
            assert launches == 1
            bound = W.wgrad_bound(self.S, self.dw0.double(), i.kb_per_split, i.splits)
            worst = R.check_out(got, want, bound, name)
            print(line + f" worst {worst:.3f}")
        return i, got


def _force_for(num_kb, kbs):
    """A YB_WGRAD_SPLITS value that gives kb_per_split == kbs, or None."""
    for n in range(1, num_kb + 1):
        if -(-num_kb // n) == kbs:
            return n
    return None


def _force_for_last(num_kb, last_of):
    """(forced count, kb_per_split) whose last split has last_of(kb_per_split) blocks and kb_per_split > 1, preferring
    the deepest such split; None if there is none."""
    for n in range(2, num_kb + 1):
        kbs = -(-num_kb // n)
        splits = -(-num_kb // kbs)
        if kbs > 1 and num_kb - (splits - 1) * kbs == last_of(kbs):
            return n, kbs
    return None


# ------------------------------------------------------------------------------------ 1. ring depth vs split count
# (name, shape (n, h, w, cin, cout, k, s), YB_WGRAD_TP, (bnw, tp)): 2 x 98 x 98 = 19208 pixels = 301 blocks, so every
# blocks-per-split value up to 17 is reachable by some forced split count.
RING = [("64x3", (2, 98, 98, 64, 128, 3, 1), None, (64, 3)),
        ("64x1", (2, 98, 98, 64, 128, 3, 1), "1", (64, 1)),
        ("32x3", (2, 98, 98, 32, 64, 3, 1), None, (32, 3)),
        ("32x1", (2, 98, 98, 32, 64, 3, 1), "1", (32, 1)),
        ("128x1", (2, 98, 98, 128, 64, 1, 1), None, (128, 1))]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_wgrad_ring_depth_vs_split_count(L, dtype):
    """Every kernel instantiation with kb_per_split = 1 .. 2 stages + 1 and num_kb (one split), a last split of one
    block and one of kb_per_split - 1: all exact, so identical across splits and YB_WGRAD_TP."""
    probs = {}
    for name, shape, tp, want in RING:
        if shape not in probs:
            probs[shape] = Problem(L, *shape, dtype=dtype, seed=11)
        p = probs[shape]
        L.set_option("YB_WGRAD_TP", tp)
        i0 = p.schedule()
        assert (i0.bnw, i0.tp) == want, name
        st, nk = i0.stages, i0.num_kb
        targets = sorted(set(range(1, 2 * st + 2)) | {nk})
        residues = set()
        for kbs in targets:
            forced = _force_for(nk, kbs)
            assert forced is not None, f"{name}: no split count gives {kbs} blocks per split"
            L.set_option("YB_WGRAD_SPLITS", forced)
            i, _ = p.check(f"{name} {dtype} kbs={kbs}")
            assert i.kb_per_split == kbs and (i.splits - 1) * kbs < nk <= i.splits * kbs
            residues.add(kbs % st)
        assert residues == set(range(st)), f"{name}: residues {sorted(residues)} of {st}"
        for what, last_of in (("last=1", lambda k: 1), ("last=kbs-1", lambda k: k - 1)):
            f = _force_for_last(nk, last_of)
            assert f is not None, f"{name}: no split count gives {what}"
            L.set_option("YB_WGRAD_SPLITS", f[0])
            i, _ = p.check(f"{name} {dtype} {what}")
            assert i.num_kb - (i.splits - 1) * i.kb_per_split == last_of(i.kb_per_split)
        L.set_option("YB_WGRAD_SPLITS", None)
        p.check(f"{name} {dtype} default")
    L.set_option("YB_WGRAD_TP", None)


# --------------------------------------------------------------------------------------------- 2. geometry edges
# (name, (n, h, w, cin, cout, k, s), extra Problem arguments); every case launches twice on a nonzero dw0
GEOMETRY = [
    ("P%64=0", (1, 16, 16, 64, 64, 3, 1), {}),
    ("P%64=1", (1, 5, 13, 32, 64, 3, 1), {}),
    ("P%64=63", (1, 9, 7, 64, 128, 3, 1), {}),
    ("P=255", (1, 15, 17, 128, 64, 1, 1), {}),
    ("13x13 images", (3, 13, 13, 64, 128, 3, 1), {}),
    ("26x26", (2, 26, 26, 128, 64, 3, 1), {}),
    ("10x22", (3, 10, 22, 32, 64, 3, 1), {}),
    ("s2 plain", (2, 26, 26, 64, 128, 3, 2), {}),
    ("s2 dilated", (2, 26, 26, 64, 128, 3, 2), {"dilated": True}),
    ("s2 dilated 20x36 cin32", (2, 20, 36, 32, 64, 3, 2), {"dilated": True}),
    ("cout32 1x1", (2, 20, 20, 64, 32, 1, 1), {}),
    ("cout32 3x3", (2, 12, 20, 32, 32, 3, 1), {}),
    ("cout64", (2, 13, 13, 128, 64, 3, 1), {}),
    ("cout255 ld256", (2, 13, 13, 256, 255, 1, 1), {"dz_ld": 256}),
    ("cout255 ld256 26", (2, 26, 26, 128, 255, 1, 1), {"dz_ld": 256}),
    ("cout1024", (1, 13, 13, 512, 1024, 3, 1), {}),
    ("cat2 slice 128 of 384", (2, 52, 52, 256, 512, 3, 2), {"in_ld": 384, "in_off": 128}),
    ("cat1 slice 256 of 768", (2, 26, 26, 512, 1024, 3, 2), {"in_ld": 768, "in_off": 256}),
    ("cat2 slice dilated", (2, 52, 52, 256, 512, 3, 2), {"in_ld": 384, "in_off": 128, "dilated": True}),
]


@pytest.mark.parametrize("name,shape,kw", GEOMETRY, ids=[g[0] for g in GEOMETRY])
def test_wgrad_geometry_exact(L, name, shape, kw):
    """Default plan (one or a few blocks per CTA: the TMA boxes cross rows and images), then one split, where the
    producer's pixel counters walk every row and image boundary; two launches accumulate dw0 + 2 ref."""
    dtype = torch.bfloat16 if sum(map(ord, name)) % 2 else torch.float16
    p = Problem(L, *shape, dtype=dtype, seed=len(name), **kw)
    p.check(f"{name} {dtype} x2", launches=2)
    L.set_option("YB_WGRAD_SPLITS", 1)
    i, _ = p.check(f"{name} {dtype} one split")
    assert i.splits == 1 and i.kb_per_split == i.num_kb


# ------------------------------------------------------------------------------------ 3. float operands, bound
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("shape,kw", [((2, 30, 34, 64, 128, 3, 1), {}), ((2, 26, 26, 128, 255, 1, 1), {"dz_ld": 256}),
                                      ((2, 28, 36, 32, 64, 3, 2), {"dilated": True})])
def test_wgrad_float_within_bound(L, shape, kw, dtype):
    p = Problem(L, *shape, dtype=dtype, exact=False, seed=5, **kw)
    nk = p.schedule().num_kb
    for forced in (None, 1, 2, 7, nk):
        L.set_option("YB_WGRAD_SPLITS", forced)
        p.check(f"float {shape} {dtype} splits={forced}")
    L.set_option("YB_WGRAD_TP", "1")
    p.check(f"float {shape} {dtype} tp1")


# ----------------------------------------------------------------------------- 4. every training layer shape
# The plan stores route 1 at channel 128 of the [52, 52, 384] concat buffer and route 2 at channel 256 of the
# [26, 26, 768] one (csrc/net.cu); the stride-2 convs that follow read their input from there.
SLICES = {(8, 256, 512): (384, 128), (16, 512, 1024): (768, 256)}     # (H / in_h, cin, cout) -> (in_ld, in_off)


def _training_shapes(L, H=416, classes=80):
    """Distinct wgrad problems of the H x H training plan (the stem excluded): (in_h, cin, cout, k, s, in_ld, in_off,
    dz_ld), from the plan's own layer table."""
    from yolov3_tensorflow_b200.model import yolov3
    table = yolov3.conv_table(classes)
    h = C.c_void_p()
    L.check(L.lib.yb_net_create(C.byref(h), classes, 1, H, H, 0, 0), "net_create")
    shapes = []
    try:
        for i in range(1, L.lib.yb_net_num_layers(h)):
            info = L.LayerInfo()
            L.check(L.lib.yb_net_layer_info(h, i, C.byref(info)), "layer_info")
            assert (info.cin, info.cout, info.ksize, info.stride, bool(info.has_bn)) == table[i]
            in_ld, in_off = SLICES.get((H // info.in_h, info.cin, info.cout), (info.cin, 0))
            dz_ld = info.cout if info.has_bn else -(-info.cout // 32) * 32
            sh = (info.in_h, info.cin, info.cout, info.ksize, info.stride, in_ld, in_off, dz_ld)
            if sh not in shapes:
                shapes.append(sh)
    finally:
        L.lib.yb_net_destroy(h)
    return shapes


def test_training_plan_has_the_expected_shapes(L):
    shapes = _training_shapes(L)
    assert 18 <= len(shapes) <= 24, len(shapes)
    assert (52, 256, 512, 3, 2, 384, 128, 512) in shapes and (26, 512, 1024, 3, 2, 768, 256, 1024) in shapes
    assert (13, 1024, 255, 1, 1, 1024, 0, 256) in shapes and (208, 64, 32, 1, 1, 64, 0, 32) in shapes
    assert (26, 768, 256, 1, 1, 768, 0, 256) in shapes and (52, 384, 128, 1, 1, 384, 0, 128) in shapes


def test_wgrad_every_training_layer_batch8(L):
    deep = 0
    for j, (hh, cin, cout, k, s, in_ld, in_off, dz_ld) in enumerate(_training_shapes(L)):
        dtype = torch.float16 if j % 2 == 0 else torch.bfloat16
        p = Problem(L, 8, hh, hh, cin, cout, k, s, dtype=dtype, in_ld=in_ld, in_off=in_off, dz_ld=dz_ld, seed=j)
        i, _ = p.check(f"layer {hh}^2 {cin}->{cout} k{k} s{s} ld {in_ld}+{in_off} dz_ld {dz_ld} b8 {dtype}")
        deep += i.kb_per_split >= 2 * i.stages
        del p
    assert deep >= 8, f"only {deep} layers wrap the ring twice at batch 8"


@pytest.mark.parametrize("n,hh,cin,cout,k,s", [(32, 416, 32, 64, 3, 2), (32, 52, 128, 256, 3, 1),
                                               (8, 608, 32, 64, 3, 2)])
def test_wgrad_deepest_loops(L, n, hh, cin, cout, k, s):
    """Layer 1 (32 -> 64, stride 2) at batch 32 (~490 blocks per CTA) and at 608 x 608, the 52 x 52 128 -> 256 3x3
    at batch 32 (~120): exact, with the default plan."""
    p = Problem(L, n, hh, hh, cin, cout, k, s, dtype=torch.float16, seed=n + hh)
    i, _ = p.check(f"deep {hh}^2 {cin}->{cout} b{n}")
    assert i.kb_per_split >= 2 * i.stages, (i.kb_per_split, i.stages)


# --------------------------------------------------------------------------------------------------- 5. stem
STEM_TH, STEM_TW = 8, 16             # stem_wgrad_tc_kernel's output tile


class StemProblem:
    def __init__(self, L, n, h, w, dtype, exact, seed=0):
        self.L, self.dtype, self.exact = L, dtype, exact
        self.n, self.h, self.w = n, h, w
        g = torch.Generator(device="cuda").manual_seed(seed)
        P = n * h * w
        if exact:
            # image k / 8 in [0, 1]; dz in {-1, 0, 1} keeps 8 S below 2^24 at batch 32 x 416^2
            self.img = _ints((n, h, w, 3), 0, 8, g).float() / 8
            self.dz = _ints((n, h, w, 32), -1, 1, g).to(dtype)
            self.dw0 = _ints((32, 27), -64, 64, g).float()
        else:
            self.img = torch.rand((n, h, w, 3), generator=g, device="cuda")
            self.dz = (torch.randn((n, h, w, 32), generator=g, device="cuda") * 0.1).to(dtype)
            self.dw0 = torch.randn((32, 27), generator=g, device="cuda")
        self.ref, self.S = W.wgrad_ref(self.img, self.dz, 3, 1)
        self.dz_abs = sum(self.dz[i].double().abs().sum((0, 1)) for i in range(n))      # [32]
        self.buf = torch.empty((34, 27), dtype=torch.float32, device="cuda")
        sms = _sms(L)
        tiles = n * -(-h // STEM_TH) * -(-w // STEM_TW)
        self.grid_tc = min(tiles, 4 * sms)
        self.tiles_per_cta = -(-tiles // self.grid_tc)
        self.min_tiles_per_cta = tiles // self.grid_tc
        self.blocks_cuda = min(-(-P // 8), 8 * sms)
        self.ppw = -(-P // (8 * self.blocks_cuda))

    def check(self, name, kernel):
        L = self.L
        self.buf.view(torch.int32).fill_(SENT_BITS)
        self.buf[1:-1] = self.dw0
        dwp = C.c_void_p(self.buf[1].data_ptr())
        if kernel == "tc":
            L.check(L.lib.yb_stem_conv_wgrad_tc(L.ptr(self.img), L.ptr(self.dz), _code(L, self.dtype), self.n, self.h,
                                                self.w, dwp, L.stream_handle()), "stem_wgrad_tc")
        else:
            L.set_option("YB_STEM_WGRAD", "cuda")
            try:
                L.check(L.lib.yb_stem_conv_wgrad(L.ptr(self.img), L.ptr(self.dz), _code(L, self.dtype), self.n, self.h,
                                                 self.w, dwp, L.stream_handle()), "stem_wgrad")
            finally:
                L.set_option("YB_STEM_WGRAD", None)
        torch.cuda.synchronize()
        bits = self.buf.view(torch.int32)
        assert bool((bits[0] == SENT_BITS).all()) and bool((bits[-1] == SENT_BITS).all()), f"{name}: stray writes"
        got = self.buf[1:-1]
        want = self.dw0.double() + self.ref
        line = (f"WGRAD stem {kernel} {name}: tiles/CTA {self.min_tiles_per_cta}-{self.tiles_per_cta} grid "
                f"{self.grid_tc if kernel == 'tc' else self.blocks_cuda}")
        if self.exact:
            assert 8 * float(self.S.max() + self.dw0.abs().max()) < W.EXACT_LIMIT, f"{name}: operands too large"
            diff = got.double() != want
            assert not bool(diff.any()), (f"{name}: {int(diff.sum())} elements differ; worst "
                                          f"{float((got.double() - want).abs().max())}")
            print(line + " exact")
        else:
            if kernel == "tc":
                bound = W.stem_tc_bound(self.S, self.dz_abs, self.dw0.double(), self.dtype, self.tiles_per_cta,
                                        self.grid_tc)
            else:
                bound = W.stem_cuda_bound(self.S, self.dw0.double(), self.ppw, self.blocks_cuda)
            worst = R.check_out(got, want, bound, name)
            print(line + f" worst {worst:.2e}")


@pytest.mark.parametrize("n,h,w", [(8, 416, 416), (32, 416, 416), (4, 300, 200)])
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "float"])
def test_stem_wgrad_many_tiles_per_cta(L, n, h, w, exact):
    """Both stem kernels with every CTA (warp) running several tiles (pixels): 416^2 at batch 8 and 32, and a size
    with partial 8 x 16 tiles in both directions."""
    for dtype in (torch.float16, torch.bfloat16):
        p = StemProblem(L, n, h, w, dtype, exact, seed=n + h + w)
        assert p.min_tiles_per_cta >= 3, (p.min_tiles_per_cta, p.grid_tc)
        assert p.ppw >= 3
        for kernel in ("tc", "cuda"):
            p.check(f"{n}x{h}x{w} {dtype}", kernel)
        del p
