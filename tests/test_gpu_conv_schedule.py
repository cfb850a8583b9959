"""The implicit-GEMM conv (csrc/conv_igemm.cu) over many work units per consumer warpgroup, against float64 references.

Most of what the ping-pong schedule adds happens from a warpgroup's second work unit on: the ring position it skips
over the other warpgroup's unit (which depends on num_kb mod stages), the tensor-core handoff between the two
warpgroups, the per-warpgroup scale / shift reloaded and the per-warpgroup statistics flushed when the n-tile changes.
A grid of min(units, SMs) CTAs gives small tests at most one unit per warpgroup, so every case here also runs with the
grid capped (YB_CONV_CTAS = 1, 2, 3, 7) and under both schedules where both are meaningful (YB_CONV_PP = 0 / 1).

Each case asserts its premise through yb_conv_schedule (which schedule runs, at least 3 units per warpgroup, num_kb mod
stages), so that a change of the selection rule fails here instead of silently making a case a duplicate.  Outputs are
checked element by element against the float64 bound of tests/conv_ref.py; guard rows before and after the output and
the columns outside the written channel slice must keep their sentinel; and since a tile's k-order does not depend on
which CTA or warpgroup runs it, every output is bit-identical across grid caps, across the two schedules and between
two runs.  Each run prints one "SCHED" line: case, schedule, units per warpgroup, num_kb mod stages, worst error as a
fraction of the bound."""
import ctypes as C

import pytest
import torch

from tests import conv_ref as R

pytestmark = pytest.mark.gpu

CAPS = (1, 2, 3, 7, None)
SENT = -7.0
GUARD = 128            # sentinel rows before and after every output: one tile
KEYS = ("YB_CONV_PP", "YB_CONV_CTAS", "YB_CONV_EG", "YB_CONV_MODE", "YB_CONV_MC", "YB_CONV_EPI")


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


def _schedule(L, d, kh=0, kw=0, stats=False):
    info = L.ConvSchedule()
    L.check(L.lib.yb_conv_schedule(C.byref(d), kh, kw, int(stats), _sms(L), C.byref(info)), "conv_schedule")
    return info


def _set(L, pp, cap):
    L.set_option("YB_CONV_PP", pp)
    L.set_option("YB_CONV_CTAS", cap)


def _premise(L, name, d, pp, cap, kh=0, kw=0, stats=False, want_pp=None, uncapped_units=False):
    """Schedule of this run; asserts the schedule the case is about and, when the grid is capped (or uncapped_units is
    set: the production shapes), at least 3 units per consumer warpgroup."""
    i = _schedule(L, d, kh, kw, stats)
    if want_pp is not None:
        assert i.pingpong == want_pp, f"{name}: expected {'ping-pong' if want_pp else 'cooperative'}"
    upw = R.units_per_warpgroup(i)
    if cap is not None or uncapped_units:
        assert upw >= 3, f"{name}: only {upw} units per warpgroup (grid {i.grid})"
    return i, upw


def _report(name, i, upw, worst):
    print(f"SCHED {name}: {'pp' if i.pingpong else 'coop'} {i.block_m}x{i.block_n}x{i.block_k} grid {i.grid} "
          f"units/wg {upw} num_kb {i.num_kb} mod stages {i.stages} = {i.num_kb % i.stages} worst {worst:.3f}")


class FwdCase:
    """One yb_conv2d_fwd problem: operands, float64 reference in the output's row layout, bound."""

    def __init__(self, L, n, h, w, cin, cout, k, s, dtype=torch.float16, in_extra=0, out_extra=0, res=None,
                 upsample=False, out_fp32=False, leaky=True, stats=False, identity=False, seed=0, dgrad=False):
        self.L, self.dtype, self.stats, self.res_mode = L, dtype, stats, res
        dev = "cuda"
        g = torch.Generator().manual_seed(seed)
        code = _code(L, dtype)
        in_ld = cin + in_extra
        self.xfull = (torch.randn((n, h, w, in_ld), generator=g) * (0.1 if dgrad else 1.0)).to(dtype).to(dev)
        in_off = in_extra // 2 // 8 * 8
        x = self.xfull[..., in_off:in_off + cin]
        self.xp = self.xfull.data_ptr() + in_off * 2
        if dgrad:
            # the dgrad conv of a stride-1 layer (cout_f = cout, cin_f = cin of the forward layer), weights from the packer
            fcin, fcout = cout, cin
            wt = (torch.randn((fcout, k, k, fcin), generator=g) * 0.05).to(dev)
            cin_pad = L.lib.yb_conv_cout_pad(fcin)
            wd = torch.empty((cin_pad, k, k, cin), dtype=dtype, device=dev)
            L.check(L.lib.yb_pack_dgrad_weights(L.ptr(wt), fcout, fcin, k, cin, cin_pad, code, L.ptr(wd),
                                                L.stream_handle()), "pack_dgrad")
            self.wp = wd
        else:
            wt = (torch.randn((cout, k, k, cin), generator=g) / (k * cin ** 0.5)).to(dev)
            cout_pad = L.lib.yb_conv_cout_pad(cout)
            self.wp = torch.zeros((cout_pad, k, k, cin), dtype=dtype, device=dev)
            L.check(L.lib.yb_pack_conv_weights(L.ptr(wt), L.YB_W_OHWI, cout, cin, k, cout_pad, code, L.ptr(self.wp),
                                               L.stream_handle()), "pack")
        cout_pad = L.lib.yb_conv_cout_pad(cout)
        if identity:
            self.sc, self.sh = torch.ones(cout_pad, device=dev), torch.zeros(cout_pad, device=dev)
        else:
            self.sc = torch.ones(cout_pad, device=dev); self.sc[:cout] = (torch.rand(cout, generator=g) + 0.5).to(dev)
            self.sh = torch.zeros(cout_pad, device=dev); self.sh[:cout] = (torch.randn(cout, generator=g) * 0.1).to(dev)
        P, Q = h // s, w // s
        up = 2 if upsample else 1
        self.rows = n * P * Q * up * up
        self.out_ld = cout + out_extra
        self.out_off = 0 if out_fp32 else out_extra // 2 // 8 * 8
        self.odt = torch.float32 if out_fp32 else dtype
        self.cout, self.cout_pad = cout, cout_pad
        self.prev = None
        if res is not None:
            self.prev = torch.randn((n * P * Q, cout), generator=g).to(dtype).to(dev)
        self.desc = L.ConvDesc(n=n, h=h, w=w, cin=cin, cout=cout, ksize=k, stride=s, in_ld=in_ld, out_ld=self.out_ld,
                               res_ld=self.out_ld if res == "inplace" else cout, dtype=code, out_fp32=int(out_fp32),
                               leaky=int(leaky), upsample2x=int(upsample))
        # ---- float64 reference
        raw, S = R.conv_raw(x, self.wp[:cout], s, k // 2)
        self.raw, self.S = raw, S
        ref = R.epilogue(raw, self.sc[:cout], self.sh[:cout], leaky, self.prev)
        bound = R.out_bound(ref, S, k * k * cin // 16, self.odt, self.sc[:cout], self.sh[:cout], self.prev)
        if upsample:
            def upx(t):
                t = t.reshape(n, P, Q, cout)
                return t.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).reshape(-1, cout)
            ref, bound = upx(ref), upx(bound)
        self.ref, self.bound = ref, bound
        self.n16 = k * k * cin // 16

    def run(self):
        L = self.L
        esz = 4 if self.odt == torch.float32 else 2
        buf = torch.full((GUARD + self.rows + GUARD, self.out_ld), SENT, dtype=self.odt, device="cuda")
        if self.res_mode == "inplace":
            buf[GUARD:GUARD + self.rows, self.out_off:self.out_off + self.cout] = self.prev
        op = buf.data_ptr() + (GUARD * self.out_ld + self.out_off) * esz
        resp = None
        if self.res_mode == "inplace":
            resp = C.c_void_p(op)
        elif self.res_mode == "sep":
            resp = L.ptr(self.prev)
        ssum = torch.zeros(self.cout_pad, device="cuda") if self.stats else None
        ssq = torch.zeros(self.cout_pad, device="cuda") if self.stats else None
        L.check(L.lib.yb_conv2d_fwd(C.byref(self.desc), C.c_void_p(self.xp), L.ptr(self.wp), L.ptr(self.sc), L.ptr(self.sh),
                                    resp, C.c_void_p(op), L.ptr(ssum), L.ptr(ssq), L.stream_handle()), "conv")
        torch.cuda.synchronize()
        return buf, ssum, ssq

    def check(self, name, buf, ssum, ssq, upw, grid):
        _guards(name, buf, self.rows, self.out_off, self.cout)
        got = buf[GUARD:GUARD + self.rows, self.out_off:self.out_off + self.cout]
        worst = R.check_out(got, self.ref, self.bound, name)
        if self.stats:
            b_sum, b_sq = R.stats_bound(self.raw, self.S, self.n16, R.stats_depth(max(upw, 1) + 1, grid))
            s_ref, q_ref = self.raw.sum(0), (self.raw * self.raw).sum(0)
            worst = max(worst, R.check_out(ssum[:self.cout], s_ref, b_sum, name + " ssum"),
                        R.check_out(ssq[:self.cout], q_ref, b_sq, name + " ssq"))
        return got.clone(), worst


def _guards(name, buf, rows, off, cout):
    assert bool((buf[:GUARD] == SENT).all()), f"{name}: wrote into the guard rows before the output"
    assert bool((buf[GUARD + rows:] == SENT).all()), f"{name}: wrote into the guard rows after the output"
    if buf.shape[1] > cout:
        mask = torch.ones(buf.shape[1], dtype=torch.bool, device=buf.device)
        mask[off:off + cout] = False
        assert bool((buf[GUARD:GUARD + rows][:, mask] == SENT).all()), f"{name}: wrote outside its channel slice"


def _sweep(L, name, case, pps, want, caps=CAPS, stats=False, kh=0, kw=0):
    """Run `case` under every (YB_CONV_PP, YB_CONV_CTAS) pair; want[pp] = the schedule that pp must select.  All
    outputs must be bit-identical, and a second run of the first configuration too."""
    first = None
    for pp in pps:
        for cap in caps:
            _set(L, pp, cap)
            i, upw = _premise(L, name, case.desc, pp, cap, kh, kw, stats, want[pp])
            buf, ssum, ssq = case.run()
            got, worst = case.check(f"{name} pp={pp} cap={cap}", buf, ssum, ssq, upw, i.grid)
            _report(f"{name} pp={pp} cap={cap}", i, upw, worst)
            if first is None:
                first = got
            else:
                assert torch.equal(got, first), f"{name} pp={pp} cap={cap}: output differs from the first run's bits"
    _set(L, pps[0], caps[0])
    buf, ssum, ssq = case.run()
    assert torch.equal(buf[GUARD:GUARD + case.rows, case.out_off:case.out_off + case.cout], first), f"{name}: rerun differs"


# ------------------------------------------------------------------------- k-depth against ring depth
# (k, cin, cout, dtype, num_kb, default schedule).  1x1 64-column tiles (stages 8): num_kb 1, 1, 3, 3, 5, 8, 9, 16;
# 3x3 128-column tiles (stages 6): 9, 18, 27; 3x3 128 x 32 (stages 8); 1x1 128-column tiles with cin 384: 6 = stages.
KDEPTH = [
    (1, 32, 64, torch.float16, 1, 1), (1, 64, 64, torch.bfloat16, 1, 1), (1, 96, 64, torch.float16, 3, 1),
    (1, 192, 64, torch.float16, 3, 1), (1, 320, 64, torch.bfloat16, 5, 1), (1, 512, 64, torch.float16, 8, 1),
    (1, 576, 64, torch.float16, 9, 1), (1, 1024, 64, torch.bfloat16, 16, 1),
    (3, 64, 128, torch.float16, 9, 1), (3, 128, 128, torch.bfloat16, 18, 1), (3, 192, 128, torch.float16, 27, 1),
    (3, 32, 128, torch.float16, 9, 1), (1, 384, 128, torch.float16, 6, 0),
]


@pytest.mark.parametrize("k,cin,cout,dtype,num_kb,pp_default", KDEPTH,
                         ids=[f"k{a[0]}-cin{a[1]}-cout{a[2]}-{str(a[3])[6:]}" for a in KDEPTH])
def test_kdepth_vs_ring(L, k, cin, cout, dtype, num_kb, pp_default):
    name = f"kdepth k{k} cin{cin} cout{cout}"
    case = FwdCase(L, 2, 52, 52, cin, cout, k, 1, dtype=dtype, seed=cin + k)
    i = _schedule(L, case.desc)
    assert (i.num_kb, i.pingpong) == (num_kb, pp_default)
    _sweep(L, name, case, ("0", "1"), {"0": 0, "1": 1})
    _set(L, None, "7")
    assert _schedule(L, case.desc).pingpong == pp_default


# ------------------------------------------------------------------------- tails
def _tail_geometry(r):
    """(n, h, w) with 42 < M / 128 < 70 full tiles and M mod 128 = r."""
    for n in (1, 2, 3):
        for h in range(24, 130):
            for w in range(24, 130):
                M = n * h * w
                if M % 128 == r and 42 * 128 < M < 70 * 128:
                    return n, h, w
    raise AssertionError(r)


TAILS = [(1, 1), (63, 3), (64, 1), (65, 3), (127, 3), (127, 1)]


@pytest.mark.parametrize("r,k", TAILS, ids=[f"mod{r}-k{k}" for r, k in TAILS])
def test_tail_rows(L, r, k):
    n, h, w = _tail_geometry(r)
    case = FwdCase(L, n, h, w, 64, 64, k, 1, dtype=torch.float16, res="sep", seed=r)
    assert (n * h * w) % 128 == r
    _sweep(L, f"tail M%128={r} k{k}", case, ("0", "1"), {"0": 0, "1": 1})


def test_tail_last_unit_on_both_warpgroups(L):
    """Across the tail cases and grid caps, the last (partial) unit falls on ping-pong warpgroup 0 in some runs and on
    warpgroup 1 in others."""
    seen = set()
    for r, k in TAILS:
        n, h, w = _tail_geometry(r)
        d = L.ConvDesc(n=n, h=h, w=w, cin=64, cout=64, ksize=k, stride=1, in_ld=64, out_ld=64, res_ld=64, dtype=L.YB_F16,
                       out_fp32=0, leaky=1, upsample2x=0)
        for cap in CAPS[:-1]:
            _set(L, "1", str(cap))
            seen.add(R.last_unit_warpgroup(_schedule(L, d)))
    assert seen == {0, 1}


# ------------------------------------------------------------------------- statistics across n-tiles
@pytest.mark.parametrize("k,cin,cout,dtype", [(1, 128, 192, torch.float16), (3, 64, 512, torch.bfloat16)],
                         ids=["1x1-cout192", "3x3-cout512"])
def test_stats_across_ntiles(L, k, cin, cout, dtype):
    """BN statistics (m-fastest unit order): each warpgroup crosses n-tiles, flushing its column sums every time."""
    case = FwdCase(L, 2, 52, 52, cin, cout, k, 1, dtype=dtype, leaky=False, stats=True, identity=True, seed=5)
    i = _schedule(L, case.desc, stats=True)
    assert i.num_n_tiles == (3 if cout == 192 else 4)
    for cap in ("1", "3"):
        _set(L, None, cap)
        j = _schedule(L, case.desc, stats=True)
        units, G = j.num_m_tiles * j.num_n_tiles, j.grid
        for wg in range(2 * G):                 # ping-pong warpgroup (b, w) runs units b + w G + 2 G j, n-tile = unit / m-tiles
            ntiles = {u // j.num_m_tiles for u in range(wg % G + (wg // G) * G, units, 2 * G)}
            assert len(ntiles) == j.num_n_tiles, f"cap {cap}: warpgroup {wg} sees n-tiles {sorted(ntiles)}"
    _sweep(L, f"stats k{k} cout{cout}", case, ("0", "1"), {"0": 0, "1": 1}, stats=True)


# ------------------------------------------------------------------------- epilogue features
EPI = [
    # id, kwargs of FwdCase
    ("3x3-slices-residual", dict(n=2, h=52, w=52, cin=128, cout=128, k=3, s=1, in_extra=64, out_extra=64, res="sep")),
    ("1x1-residual-inplace", dict(n=2, h=52, w=52, cin=128, cout=64, k=1, s=1, res="inplace", out_extra=32)),
    ("3x3-residual-inplace-bf16", dict(n=2, h=52, w=52, cin=64, cout=128, k=3, s=1, res="inplace", dtype=torch.bfloat16)),
    ("1x1-upsample-concat", dict(n=2, h=52, w=52, cin=128, cout=64, k=1, s=1, upsample=True, out_extra=128)),
    ("3x3-upsample-concat-bf16", dict(n=2, h=52, w=52, cin=64, cout=128, k=3, s=1, upsample=True, out_extra=256,
                                      dtype=torch.bfloat16)),
    ("1x1-fp32-cout18", dict(n=2, h=52, w=52, cin=256, cout=18, k=1, s=1, out_fp32=True, leaky=False, out_extra=5)),
    ("1x1-fp32-cout63", dict(n=2, h=52, w=52, cin=256, cout=63, k=1, s=1, out_fp32=True, leaky=False, out_extra=5)),
    ("3x3-s2-slices", dict(n=8, h=52, w=52, cin=64, cout=64, k=3, s=2, in_extra=32, out_extra=64)),
]


@pytest.mark.parametrize("eid,kw", EPI, ids=[e[0] for e in EPI])
def test_epilogue_features(L, eid, kw):
    case = FwdCase(L, seed=9, **kw)
    _sweep(L, f"epi {eid}", case, ("0", "1"), {"0": 0, "1": 1})


# ------------------------------------------------------------------------- dgrad
def test_dgrad_stride1_via_fwd(L):
    """Data gradient of a 3x3 stride-1 layer (64 -> 128): yb_conv2d_fwd over dz with the packer's flipped weights,
    identity scale / shift, added in place to the gradient already there (as the training plan does)."""
    case = FwdCase(L, 2, 52, 52, 128, 64, 3, 1, dtype=torch.float16, res="inplace", leaky=False, identity=True,
                   dgrad=True, seed=13)
    _sweep(L, "dgrad s1 3x3", case, ("0", "1"), {"0": 0, "1": 1})


@pytest.mark.parametrize("cin,cout,dtype", [(128, 256, torch.float16), (64, 128, torch.bfloat16)], ids=["128-256", "64-128-bf16"])
def test_dgrad_stride2_parity_classes(L, cin, cout, dtype):
    """yb_conv2d_dgrad_s2 (four parity-class window convs over the plain dz, scattered into dx and added in place)
    against float64 conv_transpose2d, with every class capped."""
    dev = "cuda"
    g = torch.Generator().manual_seed(17)
    n, h, w = 2, 104, 104
    ho, wo = h // 2, w // 2
    code = _code(L, dtype)
    wt = (torch.randn((cout, 3, 3, cin), generator=g) * 0.05).to(dev)
    kco = (cout + 31) // 32 * 32
    cin_pad = L.lib.yb_conv_cout_pad(cin)
    wd = torch.empty(9 * cin_pad * kco, dtype=dtype, device=dev)
    L.check(L.lib.yb_pack_dgrad_weights_s2(L.ptr(wt), cout, cin, kco, cin_pad, code, L.ptr(wd), L.stream_handle()), "pack_s2")
    dz = (torch.randn((n, ho, wo, kco), generator=g) * 0.1).to(dtype).to(dev)
    prev = (torch.randn((n * h * w, cin), generator=g) * 0.1).to(dtype).to(dev)
    wq = wt.to(dtype).double().permute(0, 3, 1, 2)                # OIHW of the forward conv, 16-bit-rounded
    dz64 = dz[..., :cout].double().permute(0, 3, 1, 2)
    raw = torch.nn.functional.conv_transpose2d(dz64, wq, stride=2, padding=1, output_padding=1)
    S = torch.nn.functional.conv_transpose2d(dz64.abs(), wq.abs(), stride=2, padding=1, output_padding=1)
    raw = raw.permute(0, 2, 3, 1).reshape(-1, cin)
    S = S.permute(0, 2, 3, 1).reshape(-1, cin)
    ref = raw + prev.double()
    a = (torch.arange(h, device=dev) & 1).view(1, h, 1, 1)
    b = (torch.arange(w, device=dev) & 1).view(1, 1, w, 1)
    n16 = ((1 + a) * (1 + b) * kco // 16).expand(n, h, w, 1).reshape(-1, 1).double()
    bound = R.out_bound(ref, S, n16, dtype, res=prev)
    fwd = L.ConvDesc(n=n, h=h, w=w, cin=cin, cout=cout, ksize=3, stride=2, in_ld=cin, out_ld=cout, res_ld=0, dtype=code,
                     out_fp32=0, leaky=0, upsample2x=0)
    cls = L.ConvDesc(n=n, h=ho, w=wo, cin=kco, cout=cin, ksize=1, stride=1, in_ld=kco, out_ld=cin, res_ld=cin, dtype=code,
                     out_fp32=0, leaky=0, upsample2x=0)
    rows = n * h * w
    first = None
    for pp in ("0", "1"):
        for cap in CAPS:
            _set(L, pp, cap)
            infos = []
            for c in range(4):
                i, upw = _premise(L, f"dgrad s2 class {c}", cls, pp, cap, 1 + (c >> 1), 1 + (c & 1), want_pp=int(pp))
                infos.append((i, upw))
            buf = torch.full((GUARD + rows + GUARD, cin), SENT, dtype=dtype, device=dev)
            buf[GUARD:GUARD + rows] = prev
            dx = C.c_void_p(buf.data_ptr() + GUARD * cin * 2)
            L.check(L.lib.yb_conv2d_dgrad_s2(C.byref(fwd), L.ptr(dz), kco, kco, L.ptr(wd), dx, cin, dx, cin,
                                             L.stream_handle()), "dgrad_s2")
            torch.cuda.synchronize()
            name = f"dgrad s2 {cin}->{cout} pp={pp} cap={cap}"
            _guards(name, buf, rows, 0, cin)
            got = buf[GUARD:GUARD + rows]
            worst = R.check_out(got, ref, bound, name)
            for c, (i, upw) in enumerate(infos):
                _report(f"{name} class {c}", i, upw, worst)
            if first is None:
                first = got.clone()
            else:
                assert torch.equal(got, first), f"{name}: output differs from the first run's bits"


# ------------------------------------------------------------------------- production shapes, uncapped grid
def _batch_for(L, make_desc, stats):
    """Smallest batch whose uncapped grid gives every consumer warpgroup at least 3 units on this device."""
    for n in range(1, 512):
        if R.units_per_warpgroup(_schedule(L, make_desc(n), stats=stats)) >= 3:
            return n
    raise AssertionError("no batch reaches 3 units per warpgroup")


PROD = [
    # id, (h, w, cin, cout, k, s), dtype, training forward (statistics) or inference
    ("3x3-512-1024-13-train", (13, 13, 512, 1024, 3, 1), torch.float16, True),
    ("1x1-64-32-208-train", (208, 208, 64, 32, 1, 1), torch.bfloat16, True),
    ("3x3-s2-256-512-52-infer", (52, 52, 256, 512, 3, 2), torch.float16, False),
]


@pytest.mark.parametrize("geom,dtype,train", [p[1:] for p in PROD], ids=[p[0] for p in PROD])
def test_production_shapes(L, geom, dtype, train):
    h, w, cin, cout, k, s = geom

    def desc(n):
        return L.ConvDesc(n=n, h=h, w=w, cin=cin, cout=cout, ksize=k, stride=s, in_ld=cin, out_ld=cout, res_ld=0,
                          dtype=_code(L, dtype), out_fp32=0, leaky=int(not train), upsample2x=0)
    n = _batch_for(L, desc, train)
    case = FwdCase(L, n, h, w, cin, cout, k, s, dtype=dtype, leaky=not train, stats=train, identity=train, seed=23)
    name = f"prod {h}x{w} {cin}->{cout} k{k}s{s} n{n}"
    first = None
    for rep in range(2):
        i, upw = _premise(L, name, case.desc, None, None, stats=train, want_pp=1, uncapped_units=True)
        buf, ssum, ssq = case.run()
        got, worst = case.check(name, buf, ssum, ssq, upw, i.grid)
        _report(name, i, upw, worst)
        if first is None:
            first = got
        else:
            assert torch.equal(got, first), f"{name}: rerun differs"
