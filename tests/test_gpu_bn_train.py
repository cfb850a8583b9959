"""The batch-norm training kernels (csrc/bn.cu) at every BN-layer geometry of the 416 x 416 training plan, against
float64 and exactly emulated float32 references (tests/bn_ref.py).

The streaming kernels launch one wave of SM count x blocks-per-SM blocks; a block owns rows_per_block rows, which its
row lanes walk R rows at a time (yb_bn_schedule).  Tiny tensors give every lane one row, so these tests run the real
layer sizes: batch 8 at 416 x 416 (up to 1.38 M rows), layer 0 at batch 32 (5.5 M rows) and at 608 x 608, and a
1024-channel layer at batch 32.  Each case asserts its premise through yb_bn_schedule, so a change of the launch
shape fails here instead of silently turning a case into a duplicate.

Each geometry is stored the way the plan stores it: the upsampling convs write 2x-upsampled at channel 0 of the
concat buffers (ld 768 and 384), the last residual block of stages 3 and 4 writes at channel 128 of ld 384 and 256 of
ld 768, and the backward reads dA with those strides; the stride-2 layers' dz is also stored dilated.  Everything
around an output (the other channels, GUARD rows before and after, the dilation gaps) holds nonzero poison that must
be bitwise unchanged, and every float32 output row lies between rows of -0.0, which any stray write or atomic add
changes (-0.0 + 0.0 = +0.0).

- Forward, float operands with a per-channel mean offset: finalize's mean / var / scale / shift / moving statistics bit
  for bit against float32 emulation, invstd within the rsqrtf bound, the apply output bit for bit except where the
  float64 fma emulation was inexact (one ulp then).  The fused statistics + apply launch (FIN) must equal finalize +
  apply bit for bit, for batch statistics and for frozen BN (no sums: the moving statistics stay unchanged).
- Backward, integer operands: dgamma and dbeta exact, through the workspace and through atomics, and the workspace
  all zero again after every launch; dz within the per-element bound, plain and dilated.
- Backward, float operands from the forward: dgamma / dbeta and dz within their bounds.

Each case prints one "BN" line: geometry, launch shape, and the worst error as a fraction of its bound."""
import ctypes as C

import pytest
import torch

from tests import bn_ref as B
from tests import conv_ref as R

pytestmark = pytest.mark.gpu

SENT_BITS = -(2 ** 31)            # -0.0f
EPS, DECAY = 1e-5, 0.99
GUARD = 5                         # poison rows before and after every 16-bit buffer
CHUNK = 1 << 22                   # float64 reference elements per image group

# Every distinct BN-layer geometry of the 416 x 416 training plan (csrc/net.cu Builder::build, csrc/net_train.cu):
# (name, out_h, c, residual, upsample, out_ld, out_off, stride 2)
TABLE = [
    ("416 c32 stem", 416, 32, False, False, 32, 0, False),
    ("208 c64 s2", 208, 64, False, False, 64, 0, True),
    ("208 c32", 208, 32, False, False, 32, 0, False),
    ("208 c64 res", 208, 64, True, False, 64, 0, False),
    ("104 c128 s2", 104, 128, False, False, 128, 0, True),
    ("104 c64", 104, 64, False, False, 64, 0, False),
    ("104 c128 res", 104, 128, True, False, 128, 0, False),
    ("52 c256 s2", 52, 256, False, False, 256, 0, True),
    ("52 c128", 52, 128, False, False, 128, 0, False),
    ("52 c256 res", 52, 256, True, False, 256, 0, False),
    ("52 c256 res cat2@128", 52, 256, True, False, 384, 128, False),
    ("52 c256", 52, 256, False, False, 256, 0, False),
    ("26 c512 s2", 26, 512, False, False, 512, 0, True),
    ("26 c256", 26, 256, False, False, 256, 0, False),
    ("26 c512 res", 26, 512, True, False, 512, 0, False),
    ("26 c512 res cat1@256", 26, 512, True, False, 768, 256, False),
    ("26 c512", 26, 512, False, False, 512, 0, False),
    ("26 c128 up cat2@0", 26, 128, False, True, 384, 0, False),
    ("13 c1024 s2", 13, 1024, False, False, 1024, 0, True),
    ("13 c512", 13, 512, False, False, 512, 0, False),
    ("13 c1024 res", 13, 1024, True, False, 1024, 0, False),
    ("13 c1024", 13, 1024, False, False, 1024, 0, False),
    ("13 c256 up cat1@0", 13, 256, False, True, 768, 0, False),
]


@pytest.fixture
def L():
    from yolov3_tensorflow_b200 import _lib
    _lib.set_option("YB_BN_CPT", None)
    yield _lib
    _lib.set_option("YB_BN_CPT", None)


@pytest.fixture
def ws(L):
    need = C.c_size_t()
    L.check(L.lib.yb_bn_bwd_reduce_workspace_bytes(C.byref(need)), "workspace_bytes")
    return torch.zeros(need.value, dtype=torch.uint8, device="cuda")


def _code(L, dtype):
    return L.YB_F16 if dtype == torch.float16 else L.YB_BF16


def _sms(L):
    s = C.c_int()
    L.check(L.lib.yb_device_info(C.byref(s), None, None), "device_info")
    return s.value


def schedule(L, rows, c, sms=None):
    info = L.BnSchedule()
    L.check(L.lib.yb_bn_schedule(rows, c, sms or _sms(L), C.byref(info)), "bn_schedule")
    return info


def _at(t, row, col=0):
    """Device pointer of t[row, col] of a 2-D tensor."""
    return C.c_void_p(t.data_ptr() + (row * t.shape[1] + col) * t.element_size())


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g, device="cuda", dtype=torch.int8)


def _poison(rows, ld, dtype, g):
    """[GUARD + rows + GUARD, ld] of nonzero integers."""
    v = _ints((rows + 2 * GUARD, ld), 1, 3, g)
    return torch.where(_ints(v.shape, 0, 1, g) == 0, v, -v).to(dtype)


class Sent:
    """k float32 [c] arrays, each between two rows of -0.0."""

    def __init__(self, k, c, init=None):
        self.t = torch.empty((2 * k + 1, c), dtype=torch.float32, device="cuda")
        self.t.view(torch.int32).fill_(SENT_BITS)
        for i, v in enumerate(init or ()):
            self.t[2 * i + 1] = v

    def __getitem__(self, i):
        return self.t[2 * i + 1]

    def p(self, i):
        return _at(self.t, 2 * i + 1)

    def check(self, what):
        bad = int((self.t[0::2].view(torch.int32) != SENT_BITS).sum())
        assert bad == 0, f"{what}: {bad} stray writes into the sentinel rows"


class Strided:
    """A [GUARD + n * H * W + GUARD, ld] poisoned 16-bit buffer holding an [n, h, w, c] tensor at channel `off`:
    stored plainly (H, W = h, w), 2x-upsampled (each row at its 4 places) or dilated (row (p, q) at (2p, 2q))."""

    def __init__(self, n, h, w, c, ld, off, dtype, g, mode="plain"):
        self.n, self.h, self.w, self.c, self.ld, self.off, self.mode = n, h, w, c, ld, off, mode
        k = 1 if mode == "plain" else 2
        self.H, self.W = k * h, k * w
        self.buf = _poison(n * self.H * self.W, ld, dtype, g)
        self.before = self.buf.clone()
        self.mask = torch.zeros(self.buf.shape, dtype=torch.bool, device="cuda")
        for v in self.places(self.mask, 0, n):
            v.fill_(True)

    def p(self):
        return _at(self.buf, GUARD, self.off)

    def grid(self, t, i0, i1):
        """[i1 - i0, H, W, c] view of images i0..i1 of the stored tensor (t: buf or a same-shaped tensor)."""
        per = self.H * self.W
        return t[GUARD + i0 * per:GUARD + i1 * per].view(i1 - i0, self.H, self.W, self.ld)[..., self.off:self.off + self.c]

    def places(self, t, i0, i1):
        """The views of images i0..i1 every row is stored at: 1 (plain, dilated) or 4 (upsampled) [k, h, w, c]."""
        v = self.grid(t, i0, i1)
        if self.mode == "plain":
            return [v]
        if self.mode == "dilated":
            return [v[:, 0::2, 0::2]]
        return [v[:, a::2, b::2] for a in (0, 1) for b in (0, 1)]

    def fill(self, x):
        """Store compact rows x [n * h * w, c] at every place."""
        x4 = x.view(self.n, self.h, self.w, self.c)
        for v in self.places(self.buf, 0, self.n):
            v.copy_(x4)
        self.before = self.buf.clone()

    def check_poison(self, what):
        changed = (self.buf.view(torch.int16) != self.before.view(torch.int16)) & ~self.mask
        bad = int(changed.sum())
        assert bad == 0, f"{what}: {bad} elements outside the output changed"

    def chunks(self):
        k = max(1, CHUNK // (self.h * self.w * self.c))
        for i0 in range(0, self.n, k):
            i1 = min(self.n, i0 + k)
            yield i0, i1, slice(i0 * self.h * self.w, i1 * self.h * self.w)


class Case:
    """One BN layer geometry: z [n * h * w, c] and the layer's output / dA / dz storage."""

    def __init__(self, L, n, h, c, res, up, out_ld, out_off, s2, dtype, seed, name):
        self.L, self.n, self.h, self.c, self.res, self.up = L, n, h, c, res, up
        self.out_ld, self.out_off, self.s2, self.dtype, self.name = out_ld, out_off, s2, dtype, name
        self.rows = n * h * h
        self.g = torch.Generator(device="cuda").manual_seed(seed)
        self.code = _code(L, dtype)

    def sched(self):
        return schedule(self.L, self.rows, self.c)

    def line(self, what):
        s = self.sched()
        last = self.rows - (s.grid - 1) * s.rows_per_block
        return (f"BN {self.name} n{self.n} {self.dtype} cpt {s.cpt} R {s.r} rows {self.rows} c {self.c} "
                f"ld {self.out_ld}+{self.out_off}{' up' if self.up else ''}{' res' if self.res else ''} grid {s.grid} "
                f"rows/block {s.rows_per_block} last {last} lanes {s.lanes} | {what}")

    def _out(self, mode=None):
        return Strided(self.n, self.h, self.h, self.c, self.out_ld, self.out_off, self.dtype, self.g,
                       mode or ("up" if self.up else "plain"))

    # ------------------------------------------------------------------------------------------------ forward
    def forward(self):
        L, c, rows, g = self.L, self.c, self.rows, self.g
        lib, st = L.lib, L.stream_handle
        off = torch.randn(c, generator=g, device="cuda") * 2
        std = torch.rand(c, generator=g, device="cuda") + 0.5
        z = (torch.randn((rows, c), generator=g, device="cuda") * std + off).to(self.dtype)
        res = torch.randn((rows, c), generator=g, device="cuda").to(self.dtype) if self.res else None
        zd = z.double()
        su, sq = zd.sum(0).float(), (zd * zd).sum(0).float()
        ga = torch.rand(c, generator=g, device="cuda") + 0.5
        be = torch.randn(c, generator=g, device="cuda") * 0.2
        mm0 = torch.randn(c, generator=g, device="cuda") * 0.1
        mv0 = torch.rand(c, generator=g, device="cuda") + 0.5
        self.z, self.ga = z, ga
        res_p = L.ptr(res)

        def finalize(frozen):
            co, mov = Sent(4, c), Sent(2, c, (mm0, mv0))
            L.check(lib.yb_bn_finalize(None if frozen else L.ptr(su), None if frozen else L.ptr(sq), rows, c, L.ptr(ga),
                                       L.ptr(be), EPS, DECAY, mov.p(0), mov.p(1), co.p(0), co.p(1), co.p(2), co.p(3),
                                       st()), "finalize")
            out = self._out()
            L.check(lib.yb_bn_act_apply(L.ptr(z), c, co.p(0), co.p(1), res_p, c, out.p(), self.out_ld, self.n, self.h,
                                        self.h, c, self.code, 1, int(self.up), st()), "act_apply")
            return co, mov, out

        def fin(frozen):
            co, mov = Sent(4, c), Sent(2, c, (mm0, mv0))
            out = self._out()
            L.check(lib.yb_bn_stats_act_apply(L.ptr(z), c, None if frozen else L.ptr(su), None if frozen else L.ptr(sq),
                                              L.ptr(ga), L.ptr(be), EPS, DECAY, mov.p(0), mov.p(1), co.p(0), co.p(1),
                                              co.p(2), co.p(3), res_p, c, out.p(), self.out_ld, self.n, self.h, self.h, c,
                                              self.code, 1, int(self.up), st()), "stats_act_apply")
            return co, mov, out

        soft = 0
        for frozen in (False, True):
            tag = "frozen" if frozen else "batch"
            co, mov, out = finalize(frozen)
            co2, mov2, out2 = fin(frozen)
            torch.cuda.synchronize()
            for s, what in ((co, "coefficients"), (mov, "moving statistics"), (co2, "FIN coefficients"),
                            (mov2, "FIN moving statistics")):
                s.check(f"{self.name} {tag} {what}")
            out.check_poison(f"{self.name} {tag} apply")
            out2.check_poison(f"{self.name} {tag} FIN apply")
            # FIN == finalize + apply, bit for bit (moving statistics: updated exactly once, or not at all when frozen)
            assert torch.equal(co.t.view(torch.int32), co2.t.view(torch.int32)), f"{self.name} {tag}: FIN coefficients"
            assert torch.equal(mov.t.view(torch.int32), mov2.t.view(torch.int32)), f"{self.name} {tag}: FIN moving"
            assert torch.equal(out.buf[out.mask].view(torch.int16), out2.buf[out2.mask].view(torch.int16)), \
                f"{self.name} {tag}: FIN output"
            sc, sh, smean, sinv = (co[i].cpu() for i in range(4))
            gac, bec, mm0c, mv0c = ga.cpu(), be.cpu(), mm0.cpu(), mv0.cpu()
            if frozen:
                assert B.invstd_error(mv0c, EPS, sinv) <= B.RSQRT_ULP, f"{self.name}: frozen invstd"
                assert torch.equal(sc, gac * sinv) and torch.equal(smean, mm0c), f"{self.name}: frozen scale / mean"
                assert bool(((sh.double() - (bec.double() - mm0c.double() * sc.double())).abs()
                             <= B.ulp32(sh)).all()), f"{self.name}: frozen shift"
                assert torch.equal(mov[0].cpu(), mm0c) and torch.equal(mov[1].cpu(), mv0c), f"{self.name}: frozen moved"
            else:
                mean, var, esc, esh = B.batch_coeffs(su.cpu(), sq.cpu(), rows, gac, bec, EPS, sinv)
                assert B.invstd_error(var, EPS, sinv) <= B.RSQRT_ULP, f"{self.name}: invstd beyond the rsqrtf bound"
                for got, want, what in ((smean, mean, "mean"), (sc, esc, "scale"), (sh, esh, "shift")):
                    assert torch.equal(got, want), f"{self.name}: {what} differs from the float32 emulation"
                emm, emv = B.moving_update(mm0c, mv0c, mean, var, rows, DECAY)
                assert torch.equal(mov[0].cpu(), emm) and torch.equal(mov[1].cpu(), emv), f"{self.name}: moving"
                self.coef = (co[0].clone(), co[1].clone(), co[2].clone(), co[3].clone())
            for i0, i1, rs in out.chunks():
                want, inexact = B.apply_ref(z[rs], co[0], co[1], None if res is None else res[rs], True, self.dtype)
                for v in out.places(out.buf, i0, i1):
                    soft += B.check_apply(v.reshape(-1, c), want, inexact, self.dtype, f"{self.name} {tag} apply")
        return f"fwd exact ({soft} one-ulp at inexact fma)"

    # ----------------------------------------------------------------------------------------------- backward
    def _dA(self, vals):
        """The layer-output gradient in the output's storage: vals [rows, c], or [4 rows, c] when upsampled (one
        block of rows per copy: the 4 copies of a row get different gradients)."""
        dA = self._out()
        if self.up:
            for k, v in enumerate(dA.places(dA.buf, 0, self.n)):
                v.copy_(vals[k * self.rows:(k + 1) * self.rows].view(self.n, self.h, self.h, self.c))
            dA.before = dA.buf.clone()
        else:
            dA.fill(vals)
        return dA

    def _reduce(self, dA, z, sc, sh, mu, inv, ws):
        L = self.L
        red = Sent(2, self.c)
        L.check(L.lib.yb_bn_bwd_reduce(dA.p(), self.out_ld, L.ptr(z), self.c, L.ptr(sc), L.ptr(sh), L.ptr(mu), L.ptr(inv),
                                       self.n, self.h, self.h, self.c, self.code, 1, int(self.up), red.p(0), red.p(1),
                                       L.ptr(ws), L.stream_handle()), "bwd_reduce")
        torch.cuda.synchronize()
        red.check(f"{self.name} dgamma / dbeta")
        if ws is not None:
            assert not bool(ws.any()), f"{self.name}: the workspace is not re-armed (ticket or partials nonzero)"
        return red

    def _ref_sums(self, dA, z, sc, sh, mu, inv):
        parts = []
        for i0, i1, rs in dA.chunks():
            v = dA.grid(dA.buf, i0, i1)
            dv = B.upsampled_rows(v) if self.up else v.float()
            da = B.dact(dv.reshape(-1, self.c), z[rs], sc, sh, True)
            parts.append(B.reduce_sums(da, z[rs], mu, inv))
            if self.exact_mode:
                assert bool((da == torch.round(da)).all()), f"{self.name}: dact is not integral"
        return B.reduce_ref(parts, mu, inv)

    def _bwd_apply(self, dA, z, sc, sh, mu, inv, dg, db, dilate):
        L = self.L
        dz = Strided(self.n, self.h, self.h, self.c, self.c, 0, self.dtype, self.g, "dilated" if dilate else "plain")
        L.check(L.lib.yb_bn_bwd_apply(dA.p(), self.out_ld, L.ptr(z), self.c, L.ptr(self.ga), L.ptr(sc), L.ptr(sh),
                                      L.ptr(mu), L.ptr(inv), L.ptr(dg), L.ptr(db), self.n, self.h, self.h, self.c,
                                      self.code, 1, int(self.up), int(dilate), dz.p(), self.c, L.stream_handle()),
                "bwd_apply")
        torch.cuda.synchronize()
        dz.check_poison(f"{self.name} dz{' dilated' if dilate else ''}")
        worst = 0.0
        for i0, i1, rs in dA.chunks():
            v = dA.grid(dA.buf, i0, i1)
            dv = B.upsampled_rows(v) if self.up else v.float()
            da = B.dact(dv.reshape(-1, self.c), z[rs], sc, sh, True)
            ref, bound = B.bwd_apply_ref(da, z[rs], self.ga, inv, mu, dg, db, self.rows, self.dtype)
            got = dz.places(dz.buf, i0, i1)[0].reshape(-1, self.c)
            worst = max(worst, R.check_out(got, ref, bound, f"{self.name} dz{' dilated' if dilate else ''}"))
        return worst

    def backward_exact(self, ws):
        """Integer operands: z in {-3..3}, sparse dA in 10 * {-4..4}, integer means, power-of-two invstd."""
        self.exact_mode = True
        c, rows, g = self.c, self.rows, self.g
        z = _ints((rows, c), -3, 3, g).to(self.dtype)
        sc = (torch.rand(c, generator=g, device="cuda") + 0.5) * torch.where(_ints((c,), 0, 1, g) == 0, 1.0, -1.0)
        sh = torch.randn(c, generator=g, device="cuda")
        mu = _ints((c,), -2, 2, g).float()
        inv = torch.exp2(_ints((c,), -1, 1, g).float())
        copies = 4 if self.up else 1
        # sparse dA keeps sum |dact z| + |mean| sum |dact| near 2^22 per channel at any row count
        density = min(0.5, 2.0 ** 22 / (100.0 * rows * copies))
        vals = (_ints((rows * copies, c), -4, 4, g) * 10).float()
        keep = torch.rand((rows * copies, c), generator=g, device="cuda") < density
        dA = self._dA(torch.where(keep, vals, 0.0).to(self.dtype))
        dg_ref, db_ref, G, A = self._ref_sums(dA, z, sc, sh, mu, inv)
        assert float((G + mu.double().abs() * A).max()) < B.EXACT_LIMIT, f"{self.name}: operands too large"
        got = {}
        for path, w in (("workspace", ws), ("atomic", None)):
            red = self._reduce(dA, z, sc, sh, mu, inv, w)
            for t, want, what in ((red[0], dg_ref, "dgamma"), (red[1], db_ref, "dbeta")):
                diff = t.double() != want
                if bool(diff.any()):
                    i = int(diff.nonzero()[0])
                    raise AssertionError(f"{self.name} {path}: {int(diff.sum())}/{c} {what} differ from the exact sum; "
                                         f"first channel {i}: got {float(t[i])} want {float(want[i])}")
            got[path] = red
        assert torch.equal(got["workspace"].t.view(torch.int32), got["atomic"].t.view(torch.int32))
        dg, db = got["workspace"][0], got["workspace"][1]
        worst = self._bwd_apply(dA, z, sc, sh, mu, inv, dg, db, False)
        if self.s2:
            worst = max(worst, self._bwd_apply(dA, z, sc, sh, mu, inv, dg, db, True))
        return f"bwd int: sums exact (max G {float(G.max()):.3g}), dz worst {worst:.3f}"

    def backward_float(self, ws):
        """The forward's z and coefficients, dense Gaussian dA."""
        self.exact_mode = False
        c, rows = self.c, self.rows
        sc, sh, mu, inv = self.coef
        copies = 4 if self.up else 1
        dA = self._dA((torch.randn((rows * copies, c), generator=self.g, device="cuda") * 0.1).to(self.dtype))
        dg_ref, db_ref, G, A = self._ref_sums(dA, self.z, sc, sh, mu, inv)
        red = self._reduce(dA, self.z, sc, sh, mu, inv, ws)
        s = self.sched()
        bg, bb = B.reduce_bound(G, A, mu, inv, s.rows_per_block, s.lanes, s.grid)
        wg = R.check_out(red[0], dg_ref, bg, f"{self.name} float dgamma")
        wb = R.check_out(red[1], db_ref, bb, f"{self.name} float dbeta")
        wz = self._bwd_apply(dA, self.z, sc, sh, mu, inv, red[0].clone(), red[1].clone(), self.s2)
        return f"bwd float: dgamma {wg:.3f} dbeta {wb:.3f} dz {wz:.3f}"

    def run(self, ws):
        parts = [self.forward(), self.backward_exact(ws), self.backward_float(ws)]
        print(self.line(" | ".join(parts)))


def _premises(s, rows):
    last = rows - (s.grid - 1) * s.rows_per_block
    return {"groups": -(-s.rows_per_block // s.lanes) > s.r,                # the R-row loop past its first group
            "short last block": last < s.rows_per_block,
            "tail inside an R-group": (last % s.lanes != 0) or ((last // s.lanes) % s.r != 0),
            ">= 16 blocks per slot": s.grid >= 16 * B.BN_SLOTS}


# ------------------------------------------------------------------------------------- 1. the training plan's table
def test_table_matches_the_training_plan(L):
    """TABLE == the BN layers of a bound 416 x 416 training plan: output size, channels, residual (the 3 x 3 convs of
    the residual blocks), upsample, and the dA storage (ld, channel offset) that yb_net_train_buffer reports."""
    from yolov3_tensorflow_b200.model import yolov3
    h = C.c_void_p()
    L.check(L.lib.yb_net_create(C.byref(h), 80, 1, 416, 416, L.YB_BF16, 1), "net_create")
    try:
        a, p = C.c_size_t(), C.c_size_t()
        L.check(L.lib.yb_net_arena_bytes(h, C.byref(a), C.byref(p)), "arena_bytes")
        act = torch.zeros(a.value, dtype=torch.uint8, device="cuda")
        par = torch.zeros(p.value, dtype=torch.uint8, device="cuda")
        L.check(L.lib.yb_net_bind(h, L.ptr(act), a.value, L.ptr(par), p.value, L.stream_handle()), "net_bind")
        table = yolov3.conv_table(80)
        rows = []
        for i in range(L.lib.yb_net_num_layers(h)):
            info = L.LayerInfo()
            L.check(L.lib.yb_net_layer_info(h, i, C.byref(info)), "layer_info")
            if not info.has_bn:
                continue
            assert (info.cin, info.cout, info.ksize, info.stride, True) == table[i]
            q, ld, hh, ww = C.c_void_p(), C.c_int(), C.c_int(), C.c_int()
            L.check(L.lib.yb_net_train_buffer(h, i, 2, C.byref(q), C.byref(ld), C.byref(hh), C.byref(ww)), "dA")
            assert (hh.value, ww.value) == ((2 if info.upsample2x else 1) * info.out_h,) * 2
            for which in (0, 1):       # z and dz: compact, ld = cout
                q2, ld2 = C.c_void_p(), C.c_int()
                L.check(L.lib.yb_net_train_buffer(h, i, which, C.byref(q2), C.byref(ld2), None, None), "z / dz")
                assert ld2.value == info.cout
            res = info.ksize == 3 and info.stride == 1 and not info.is_head and i > 0
            rows.append([info.out_h, info.cout, res, bool(info.upsample2x), ld.value, q.value, info.stride == 2])
        # channel offset inside a shared (concat) buffer: from the lowest dA pointer of the layers storing with that ld
        base = {r[4]: min(s[5] for s in rows if s[4] == r[4] and s[4] != s[1]) for r in rows if r[4] != r[1]}
        plan = {tuple(r[:5] + [(r[5] - base[r[4]]) // 2 if r[4] != r[1] else 0] + r[6:]) for r in rows}
        assert len(rows) == 72
        assert plan == {t[1:] for t in TABLE}, (sorted(plan - {t[1:] for t in TABLE}),
                                               sorted({t[1:] for t in TABLE} - plan))
    finally:
        L.lib.yb_net_destroy(h)


def test_table_covers_the_launch_shapes(L):
    """At batch 8 the table runs the R-row loop past its first group, short last blocks, row tails inside an R-group
    and >= 16 blocks per workspace slot, in both kernel builds."""
    for cpt in ("8", "4"):
        L.set_option("YB_BN_CPT", None if cpt == "8" else cpt)
        seen = {}
        for name, h, c, *_ in TABLE:
            s = schedule(L, 8 * h * h, c)
            assert s.cpt == int(cpt), (name, s.cpt)
            for k, v in _premises(s, 8 * h * h).items():
                seen[k] = seen.get(k, 0) + v
        print(f"BN schedule cpt {cpt}: {seen}")
        assert all(v >= 2 for v in seen.values()), seen


# --------------------------------------------------------------------------------------- 2. every geometry, batch 8
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("entry", TABLE, ids=[t[0] for t in TABLE])
def test_bn_layer_batch8(L, ws, entry, dtype):
    name, h, c, res, up, out_ld, out_off, s2 = entry
    for cpt in (8, 4):
        L.set_option("YB_BN_CPT", None if cpt == 8 else "4")
        case = Case(L, 8, h, c, res, up, out_ld, out_off, s2, dtype, seed=h * 7 + c + cpt, name=name)
        assert case.sched().cpt == cpt
        case.run(ws)
        del case


# --------------------------------------------------------------------------------------------- 3. the largest layers
@pytest.mark.parametrize("n,h,c,dtype", [(32, 416, 32, torch.bfloat16), (8, 608, 32, torch.float16),
                                         (32, 13, 1024, torch.bfloat16)], ids=["416x32 b32", "608 b8", "13 c1024 b32"])
def test_bn_large_rows(L, ws, n, h, c, dtype):
    """Layer 0 at batch 32 (5.5 M rows, 354 MB of z in bf16) and at 608 x 608, a 1024-channel layer at batch 32."""
    case = Case(L, n, h, c, False, False, c, 0, c == 1024, dtype, seed=n + h, name=f"large {h}^2 c{c}")
    s = case.sched()
    p = _premises(s, case.rows)
    if c == 32:
        assert p["groups"] and p[">= 16 blocks per slot"], p
    case.run(ws)


# ----------------------------------------------------------------------------------------- 4. workspace re-arming
def test_workspace_rearms_across_channel_counts(L, ws):
    """One workspace through c = 1024 -> 32 -> 1024 -> 32: exact sums and an all-zero workspace after every launch."""
    cases = [Case(L, 8, 13, 1024, False, False, 1024, 0, False, torch.float16, seed=1, name="ws c1024"),
             Case(L, 8, 52, 32, False, False, 32, 0, False, torch.float16, seed=2, name="ws c32")]
    for case in cases + cases:
        case.forward()
        print(case.line(case.backward_exact(ws)))


# ------------------------------------------------------------------------------------------------ 5. col_sum / stats
@pytest.mark.parametrize("hh", [13, 26, 52])
def test_col_sum_heads_exact(L, hh):
    """Bias gradient of the detection convs: dz [8 * hh^2, 256] with c = 255 (column 255 holds poison), exact."""
    g = torch.Generator(device="cuda").manual_seed(hh)
    rows = 8 * hh * hh
    x = _poison(rows, 256, torch.bfloat16, g)
    x[GUARD:GUARD + rows, :255] = _ints((rows, 255), -3, 3, g).to(torch.bfloat16)
    want = x[GUARD:GUARD + rows, :255].double()
    out = Sent(2, 255)
    L.check(L.lib.yb_col_sum(_at(x, GUARD), 256, rows, 255, L.YB_BF16, out.p(0), L.stream_handle()), "col_sum")
    torch.cuda.synchronize()
    out.check("col_sum")
    assert torch.equal(out[0].double(), want.sum(0)), "col_sum"
    assert bool((out[1].view(torch.int32) == SENT_BITS).all()), "col_sum wrote the sum of squares"
    L.check(L.lib.yb_col_stats(_at(x, GUARD), 256, rows, 255, L.YB_BF16, out.p(0), out.p(1), L.stream_handle()),
            "col_stats")
    torch.cuda.synchronize()
    out.check("col_stats")
    assert torch.equal(out[0].double(), want.sum(0)) and torch.equal(out[1].double(), (want * want).sum(0))
    print(f"BN col_sum {hh}^2 x 255 ld 256: exact")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_col_stats_stem_exact(L, dtype):
    """The stem's batch statistics on the YB_STEM_TRAIN=cuda path: yb_col_stats over 32 x 416^2 rows of 32 channels,
    values in {-1, 0, 1} (every sum below 2^24), exact."""
    g = torch.Generator(device="cuda").manual_seed(3)
    rows = 32 * 416 * 416
    x = _ints((rows, 32), -1, 1, g).to(dtype)
    out = Sent(2, 32)
    L.check(L.lib.yb_col_stats(L.ptr(x), 32, rows, 32, _code(L, dtype), out.p(0), out.p(1), L.stream_handle()),
            "col_stats")
    torch.cuda.synchronize()
    out.check("col_stats")
    xd = x.double()
    assert torch.equal(out[0].double(), xd.sum(0)) and torch.equal(out[1].double(), (xd * xd).sum(0))
    print(f"BN col_stats stem 32x416^2 x 32 {dtype}: exact")
