"""Calibrated fp8 (e4m3) inference on the H100: weight packing, the e4m3 implicit-GEMM conv, calibration, the e4m3
network plan against a fake-quantized oracle, and the yolov3.quantize_fp8() API.

Numbers every network run measures (logit, box, confidence and probability errors against the fake-quantized oracle,
and the distance to the fp16 engine, which measures the quantization itself) are merged into the JSON file named by
$YB_FP8_RECORD; nothing is written without it."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from oracle import yolov3_oracle as O
from tests import conv_ref as R
from tests import fp8_ref as F
from tests.synth import gen_inputs

pytestmark = pytest.mark.gpu

KEYS = ("YB_CONV_PP", "YB_CONV_CTAS", "YB_CONV_EG", "YB_CONV_MODE", "YB_CONV_MC", "YB_CONV_EPI")
VARIANTS = [(pp, cap) for pp in ("0", "1") for cap in (1, 3, None)]
GUARD = 128
SENT = 0x55


@pytest.fixture
def L():
    from yolov3_tensorflow_b200 import _lib
    for k in KEYS:
        _lib.set_option(k, None)
    yield _lib
    for k in KEYS:
        _lib.set_option(k, None)


def _record(name, payload):
    path = os.environ.get("YB_FP8_RECORD")
    if not path:
        return
    data = {}
    if os.path.exists(path):
        with open(path) as f:
            data = json.load(f)
    data[name] = payload
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


# ------------------------------------------------------------------------- weight packing
@pytest.mark.parametrize("layout", ["HWIO", "OIHW"])
def test_pack_weights_e4m3_bit_exact(L, layout):
    """Per-output-channel scale amax / 448 (1 for a zero row and the padding rows), RN-satfinite codes of w / scale:
    bit-exact against torch on the CPU."""
    cout, cin, k = 255, 64, 3
    g = torch.Generator().manual_seed(3)
    w = torch.randn(cout, k, k, cin, generator=g) * torch.exp2(torch.randint(-12, 4, (cout, 1, 1, 1), generator=g).float())
    w[7] = 0.0                                                     # an all-zero row
    w[9, 0, 0, 0] = 1e-30                                          # a row whose codes are mostly zero
    src = w.permute(1, 2, 3, 0) if layout == "HWIO" else w.permute(0, 3, 1, 2)
    code = L.YB_W_HWIO if layout == "HWIO" else L.YB_W_OIHW
    cp = L.lib.yb_conv_cout_pad(cout)
    K = k * k * cin
    dst = torch.full((cp, K), 0xAB, dtype=torch.uint8, device="cuda")
    sc = torch.full((cp,), -1.0, device="cuda")
    L.check(L.lib.yb_pack_conv_weights_e4m3(L.ptr(src.contiguous().cuda()), code, cout, cin, k, cp, L.ptr(dst), L.ptr(sc),
                                            None), "pack_e4m3")
    torch.cuda.synchronize()
    wm = w.reshape(cout, K)
    amax = wm.abs().amax(1)
    s = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    q = (wm / s[:, None]).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
    want_q = torch.zeros(cp, K, dtype=torch.uint8)
    want_q[:cout] = q
    want_s = torch.ones(cp)
    want_s[:cout] = s
    assert torch.equal(sc.cpu(), want_s)
    assert torch.equal(dst.cpu(), want_q)
    assert bool((dst[7] == 0).all()) and float(sc[7]) == 1.0 and float(sc[255]) == 1.0


# ------------------------------------------------------------------------- calibration reduction
@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_amax_exact(L, dt):
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(3001, 200, generator=g) * 7).to(dt).cuda()
    out = torch.empty(1, device="cuda")
    code = L.YB_F16 if dt == torch.float16 else L.YB_BF16
    L.check(L.lib.yb_amax(L.ptr(x[:, 8:]), 200, 3001, 150, code, L.ptr(out), None), "amax")
    assert float(out) == float(x[:, 8:158].abs().max().float())


# ------------------------------------------------------------------------- the e4m3 conv
class Case:
    def __init__(self, name, n, h, w, cin, cout, k=1, s=1, in_ld=None, res=False, up=False, fp32=False, out_ld=None,
                 out_off=0):
        self.__dict__.update(name=name, n=n, h=h, w=w, cin=cin, cout=cout, k=k, s=s, in_ld=in_ld or cin, res=res, up=up,
                             fp32=fp32, out_ld=out_ld or cout, out_off=out_off)


CASES = [
    Case("1x1 128->64 (64-col tile, M tail)", 1, 20, 20, 128, 64),
    Case("1x1 256->128 (128-col tile, M tail)", 2, 18, 14, 256, 128),
    Case("3x3/1 128->128", 2, 16, 12, 128, 128, k=3),
    Case("3x3/1 256->256", 1, 12, 16, 256, 256, k=3),
    Case("3x3/2 64->128 (64-byte rows)", 2, 24, 20, 64, 128, k=3, s=2),
    Case("3x3/1 128->256 + residual", 2, 10, 14, 128, 256, k=3, res=True),
    Case("1x1 256->128 upsample into concat slice", 2, 9, 7, 256, 128, up=True, out_ld=384, out_off=0),
    Case("1x1 128->64 strided input", 2, 13, 11, 128, 64, in_ld=384),
    Case("1x1 256->255 fp32 head", 2, 13, 13, 256, 255, fp32=True),
    Case("1x1 128->63 fp32 head", 1, 26, 20, 128, 63, fp32=True),
]


def _desc(L, c):
    d = L.ConvDesc()
    d.n, d.h, d.w, d.cin, d.cout, d.ksize, d.stride = c.n, c.h, c.w, c.cin, c.cout, c.k, c.s
    d.in_ld, d.out_ld, d.res_ld = c.in_ld, c.out_ld, c.cout if c.res else 0
    d.dtype, d.out_fp32, d.leaky, d.upsample2x = L.YB_E4M3, int(c.fp32), int(not c.fp32), int(c.up)
    return d


def _setup(L, c, seed):
    g = torch.Generator().manual_seed(seed)
    P, Q = c.h // c.s, c.w // c.s
    M = c.n * P * Q
    x = F.to_codes((torch.randn(c.n, c.h, c.w, c.in_ld, generator=g) * 3).clamp(-448, 448))
    w = torch.randn(c.cout, c.k, c.k, c.cin, generator=g) * (1.0 + torch.rand(c.cout, 1, 1, 1, generator=g))
    cp = L.lib.yb_conv_cout_pad(c.cout)
    K = c.k * c.k * c.cin
    wq = torch.empty(cp, K, dtype=torch.uint8, device="cuda")
    ws = torch.empty(cp, device="cuda")
    L.check(L.lib.yb_pack_conv_weights_e4m3(L.ptr(w.cuda()), L.YB_W_OHWI, c.cout, c.cin, c.k, cp, L.ptr(wq), L.ptr(ws), None),
            "pack")
    s_in = 0.05
    scale = ((0.5 + torch.rand(cp, generator=g)) * s_in * ws.cpu()).float()
    shift = (torch.randn(cp, generator=g) * 0.5).float()
    res = F.to_codes((torch.randn(M, c.cout, generator=g) * 4).clamp(-448, 448)) if c.res else None
    res_scale = 0.03
    # float64 reference on the same codes
    xc = F.from_codes(x)[..., : c.cin]
    wc = F.from_codes(wq.cpu())[: c.cout].reshape(c.cout, c.k, c.k, c.cin)
    raw, S = R.conv_raw(xc, wc, c.s, c.k // 2)
    v = raw * scale[: c.cout].double() + shift[: c.cout].double()
    if not c.fp32:
        v = torch.where(v > 0, v, R.SLOPE * v)
    if c.res:
        v = v + F.from_codes(res) * res_scale
    bound = F.fp8_bound(S, K // 32, scale[: c.cout], shift[: c.cout], None if res is None else F.from_codes(res), res_scale)
    s_out = float(np.float32(float(v.abs().max()) / 300.0))
    return dict(x=x.cuda(), wq=wq, scale=scale.cuda(), shift=shift.cuda(), res=None if res is None else res.cuda(),
                res_scale=res_scale, s_out=s_out, ref=v, bound=bound, M=M, P=P, Q=Q)


def _out_rows(c, t):
    return t["M"] * (4 if c.up else 1)


def _run(L, c, t):
    rows = _out_rows(c, t)
    if c.fp32:
        out = torch.full(((rows + 2 * GUARD), c.out_ld), -7.0, device="cuda")
    else:
        out = torch.full(((rows + 2 * GUARD), c.out_ld), SENT, dtype=torch.uint8, device="cuda")
    d = _desc(L, c)
    view = out[GUARD:]
    optr = C.c_void_p(view.data_ptr() + c.out_off * view.element_size())
    L.check(L.lib.yb_conv2d_fwd_e4m3(C.byref(d), L.ptr(t["x"]), L.ptr(t["wq"]), L.ptr(t["scale"]), L.ptr(t["shift"]),
                                     L.ptr(t["res"]), t["res_scale"], optr, t["s_out"], None), "conv_e4m3")
    torch.cuda.synchronize()
    return out


def _expected_rows(c, t, v):
    """[M, cout] in (n, p, q) order -> the output buffer's row order (upsample: 4 copies per pixel)."""
    if not c.up:
        return v
    n, P, Q = c.n, t["P"], t["Q"]
    v = v.reshape(n, P, Q, -1).repeat_interleave(2, 1).repeat_interleave(2, 2)
    return v.reshape(n * 4 * P * Q, -1)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_conv_e4m3(L, case):
    """Every schedule (YB_CONV_PP 0 / 1) and grid cap (1, 3, uncapped) gives the same bits, twice in a row; outputs
    are within one e4m3 ulp of RN(ref) and equal to it away from rounding midpoints (fp32 heads: within the bound);
    guard rows and the columns outside the written slice keep their sentinel."""
    c = case
    t = _setup(L, c, seed=CASES.index(c))
    rows = _out_rows(c, t)
    first = None
    for pp, cap in VARIANTS:
        L.set_option("YB_CONV_PP", pp)
        L.set_option("YB_CONV_CTAS", cap)
        info = L.ConvSchedule()
        s = C.c_int()
        L.check(L.lib.yb_device_info(C.byref(s), None, None), "device_info")
        d = _desc(L, c)
        L.check(L.lib.yb_conv_schedule(C.byref(d), 0, 0, 0, s.value, C.byref(info)), "schedule")
        assert info.pingpong == int(pp) and info.block_k == (128 if c.cin % 128 == 0 else 64)
        out = _run(L, c, t)
        if first is None:
            first = out
            again = _run(L, c, t)
            assert torch.equal(again, first), f"{c.name}: two runs differ"
        else:
            assert torch.equal(out, first), f"{c.name}: PP={pp} CTAS={cap} differs from PP=0 CTAS=1"
    o = first.cpu()
    sent = -7.0 if c.fp32 else SENT
    assert bool((o[:GUARD] == sent).all()) and bool((o[GUARD + rows:] == sent).all()), f"{c.name}: guard rows written"
    body = o[GUARD: GUARD + rows]
    lo, hi = c.out_off, c.out_off + c.cout
    assert bool((body[:, :lo] == sent).all()) and bool((body[:, hi:] == sent).all()), f"{c.name}: columns outside the slice"
    ref = _expected_rows(c, t, t["ref"])
    bound = _expected_rows(c, t, t["bound"])
    if c.fp32:
        worst = R.check_out(body[:, lo:hi].double(), ref, bound, c.name)
        print(f"FP8CONV {c.name}: fp32 worst err/bound {worst:.3f}")
    else:
        inv = float(np.float32(1.0 / np.float32(t["s_out"])))
        exact, worst_ulp, n_far = F.check_e4m3(body[:, lo:hi].contiguous(), ref * inv, bound * inv, c.name)
        print(f"FP8CONV {c.name}: exact-checked fraction {exact:.4f}, worst {worst_ulp:.2f} ulp, "
              f"{n_far} near-zero outputs within one ulp + bound")


@pytest.mark.parametrize("key,val", [("YB_CONV_MODE", "2cta"), ("YB_CONV_EPI", "reg"), ("YB_CONV_EG", "1")])
def test_conv_e4m3_rejects_16bit_only_variants(L, key, val):
    c = CASES[0]
    t = _setup(L, c, seed=1)
    L.set_option(key, val)
    d = _desc(L, c)
    out = torch.empty(t["M"], c.out_ld, dtype=torch.uint8, device="cuda")
    rc = L.lib.yb_conv2d_fwd_e4m3(C.byref(d), L.ptr(t["x"]), L.ptr(t["wq"]), L.ptr(t["scale"]), L.ptr(t["shift"]), None,
                                  1.0, L.ptr(out), 1.0, None)
    assert rc == -1, f"{key}={val} accepted for e4m3"


# ------------------------------------------------------------------------- network
CONCATS = ((59, 42), (67, 25))      # (upsampling conv, route conv) writing the two concat buffers


def _params(weights, cn=80):
    if weights == "cfg1":
        return O.make_params(cn, seed=7)
    return O.make_params(cn, seed=7, random_bn=True, det_scale=8.0, conf_bias=-2.0)


def _models(weights, calib, cn=80):
    import yolov3_tensorflow_b200 as pkg
    m = pkg.yolov3(cn, O.COCO_ANCHORS, dtype="fp16")
    m.set_params(_params(weights, cn), "HWIO")
    qm = m.quantize_fp8([torch.from_numpy(b).cuda() for b in calib])
    return m, qm


_CACHE = {}


def _cached_models(weights):
    if weights not in _CACHE:
        x = gen_inputs(31, 2, 416, 416)
        _CACHE[weights] = (x,) + _models(weights, [x])
    return _CACHE[weights]


def test_calibration_amax_and_buffer_scales():
    """Each layer's amax is abs().max() of the fp16 plan's layer output (maxed over the calibration batches); each e4m3
    buffer's scale is max(amax of its producers) / 448, and both concat buffers cover both of their producers."""
    import yolov3_tensorflow_b200 as pkg
    b1, b2 = gen_inputs(41, 2, 128, 160), gen_inputs(42, 2, 128, 160)
    m = pkg.yolov3(80, O.COCO_ANCHORS, dtype="fp16")
    m.set_params(_params("cfg2"), "HWIO")
    per = []
    for b in (b1, b2):
        m.forward(torch.from_numpy(b).cuda())
        pl = m._last_plan
        per.append([float(pl.layer_output(i).abs().max()) if (i > 0 and pl.layer_info(i).has_bn) else 0.0
                    for i in range(75)])
    want = np.maximum(np.array(per[0], np.float32), np.array(per[1], np.float32))
    qm = m.quantize_fp8([torch.from_numpy(b1).cuda(), torch.from_numpy(b2).cuda()])
    assert np.array_equal(np.array(qm._fp8_amax, np.float32), want)
    qm.forward(torch.from_numpy(b1).cuda())
    sc = qm.fp8_scales()
    act = sc["act"]
    producers = {i: [i] for i in range(75)}
    for up, route in CONCATS:
        assert qm._last_plan.layer_info(up).upsample2x == 1
        producers[up] = producers[route] = [up, route]
    for i in range(3, 75):
        info = qm._last_plan.layer_info(i)
        if not info.has_bn:
            assert act[i][2] == 1.0
            continue
        mx = np.float32(max(want[j] for j in producers[i]))
        assert act[i][2] == float(mx / np.float32(448.0) if mx > 0 else np.float32(1.0)), i
        assert (sc["weight"][i] is None) == (i < 4)
    for up, route in CONCATS:
        assert act[up][2] == act[route][2]
    for i in range(0, 3):
        assert act[i][2] == 1.0                                   # fp16 buffers


class _FQNet(O._Net):
    """The oracle's inference forward with the fp8 plan's quantization points: layers 0-2 store fp16, layers >= 3 store
    e4m3 with the engine's buffer scales, layers >= 4 use per-output-channel e4m3 weights, heads are float32.
    forced: {layer: the engine's output of that layer (NCHW; e4m3 layers: codes as floats, fp16 layers: values)}: each
    such layer's output is checked against the oracle's value and its bound (tests/fp8_ref.py, tests/conv_ref.py) and the
    engine's is passed on, so every layer is checked on the engine's own inputs (results in self.cmp)."""

    def __init__(self, params, s_out, w_scale, forced=None):
        super().__init__(params, False, "fp16", 0.999, torch.float32, None)
        self.s_out, self.w_scale = s_out, w_scale
        self.forced, self.cmp, self.head_bounds = forced or {}, {}, []

    def conv2d(self, x, filters, k, strides=1, bn=True, shortcut=None):
        i = self.i
        v, bound = self._conv2d(x, filters, k, strides, bn, shortcut)   # float64 value before the store, and its bound
        if not bn:
            self.head_bounds.append(bound)
            return v.float()
        if i < 3:
            y = O._round_store(v.float(), "fp16")
        else:
            inv = float(np.float32(1.0 / np.float32(self.s_out[i])))
            y = (F.e4m3_round(v * inv) * self.s_out[i]).float()
        e = self.forced.get(i)
        if e is None:
            return y
        if i >= 3:                          # the engine's e4m3 codes against RN(value / s_out)
            exact, worst, near0 = F.check_e4m3(F.to_codes(e), v * inv, bound * inv, f"layer {i}")
            self.cmp[i] = {"exact_checked": exact, "worst_ulps": worst, "near_zero_beyond_one_ulp": near0}
            return (e.double() * self.s_out[i]).float()
        b16 = bound + 0.5 * R.ulp(v.abs() + bound, torch.float16)
        self.cmp[i] = {"worst_err_over_bound": R.check_out(e, v, b16, f"layer {i}")}
        return e

    def _conv2d(self, x, filters, k, strides, bn, shortcut):
        i = self.i
        p = self.p[i]
        self.i += 1
        w = self._t(p["w"])
        if i >= 4:
            s = self.w_scale[i][:filters].float()
            w = (F.e4m3_round(w / s) * s.double()).float()        # HWIO: the output channel is the last axis
        else:
            w = O._round_store(w, "fp16")
        wt = w.permute(3, 2, 0, 1).double()
        v = TF.conv2d(x.double(), wt, None, stride=strides, padding=k // 2)
        S = TF.conv2d(x.double().abs(), wt.abs(), None, stride=strides, padding=k // 2) if self.forced else 0.0
        if bn:
            mean, var = self._t(p["mean"]), self._t(p["var"])
            scale = self._t(p["gamma"]) / torch.sqrt(var + 1e-5)
            shift = self._t(p["beta"]) - mean * scale
            sc, sh = scale.double().view(1, -1, 1, 1), shift.double().view(1, -1, 1, 1)
            v = v * sc + sh
            v = torch.where(v > 0, v, R.SLOPE * v)
        else:
            sc, sh = 1.0, self._t(p["b"]).double().view(1, -1, 1, 1)
            v = v + sh
        r = 0.0
        if shortcut is not None:
            v = v + shortcut.double()
            r = shortcut.double().abs()
        n32 = k * k * x.shape[1] / 32
        sca = sc.abs() if bn else 1.0
        bound = F.C_STEP8 * n32 * sca * S + 4 * F.U32 * (sca * S + sh.abs() + r)
        return v, bound


def fq_forward(x, params, s_out, w_scale, forced=None, cmp=None):
    net = _FQNet(params, s_out, w_scale, forced)
    t = O._round_store(torch.from_numpy(x), "fp16").permute(0, 3, 1, 2)
    r1, r2, r3 = net.darknet53_body(t)
    i1, n1 = net.yolo_block(r3, 512)
    fm1 = net.conv2d(n1, 255, 1, bn=False)
    i1 = net.upsample(net.conv2d(i1, 256, 1), r2.shape[2:])
    i2, n2 = net.yolo_block(torch.cat([i1, r2], 1), 256)
    fm2 = net.conv2d(n2, 255, 1, bn=False)
    i2 = net.upsample(net.conv2d(i2, 128, 1), r1.shape[2:])
    _, n3 = net.yolo_block(torch.cat([i2, r1], 1), 128)
    fm3 = net.conv2d(n3, 255, 1, bn=False)
    if cmp is not None:
        cmp.update(net.cmp)
        cmp["head_bounds"] = [b.permute(0, 2, 3, 1).contiguous() for b in net.head_bounds]
    return [f.permute(0, 2, 3, 1).contiguous().numpy() for f in (fm1, fm2, fm3)]


def _err(a, b, floor):
    e = np.abs(a.astype(np.float64) - b.astype(np.float64)) / np.maximum(np.abs(b.astype(np.float64)), floor)
    return {"max": float(e.max()), "p999": float(np.quantile(e, 0.999)), "mean": float(e.mean())}


def _compare(got_f, ref_f, size):
    r = {}
    for name, a, ref in zip(("fm1", "fm2", "fm3"), got_f, ref_f):
        r[name + "_maxnorm"] = float(np.max(np.abs(a - ref)) / max(np.max(np.abs(ref)), 1e-6))
    with np.errstate(over="ignore"):
        gb, gc, gp = O.predict(got_f, O.COCO_ANCHORS, (size, size), 80)
        rb, rc, rp = O.predict(ref_f, O.COCO_ANCHORS, (size, size), 80)
    ok = np.concatenate([(np.abs(f.reshape(f.shape[0], -1, 3, 85)[..., 2:4]) < 4.0).all(-1).reshape(f.shape[0], -1)
                         for f in ref_f], axis=1)
    r["boxes"] = _err(gb[ok], rb[ok], 16.0)
    r["confs"] = _err(gc, rc, 1e-2)
    r["probs"] = _err(gp, rp, 1e-2)
    return r


def _engine_outputs(qm):
    """{layer: the quantized model's output of that layer, NCHW} for the BN layers >= 1 (layer 0's output is
    never written: the stem is fused into Conv_1); the upsampling convs' outputs are taken before the upsample."""
    pl = qm._last_plan
    out = {}
    for i in range(1, pl.num_layers):
        info = pl.layer_info(i)
        if not info.has_bn:
            continue
        y = pl.layer_output(i).float()                  # e4m3 layers: the codes' values (the oracle applies s_out)
        if info.upsample2x:
            y = y[:, ::2, ::2]
        out[i] = y.permute(0, 3, 1, 2).contiguous().cpu()
    return out


@pytest.mark.parametrize("weights", ["cfg1", "cfg2"])
def test_network_layers_vs_fake_quant_oracle(weights):
    """Layer by layer on the engine's own inputs (teacher forcing), at 416 x 416, batch 2: every e4m3 layer meets the
    criteria of the e4m3 conv unit tests (tests/fp8_ref.py) against a float64 oracle that quantizes at the same points,
    the fp16 layers 1-2 and the float32 detection heads are within their bounds."""
    x, m, qm = _cached_models(weights)
    fms = [f.cpu() for f in qm.forward(torch.from_numpy(x).cuda())]
    sc = qm.fp8_scales()
    cmp = {}
    ref = fq_forward(x, _params(weights), [a[2] for a in sc["act"]], sc["weight"], _engine_outputs(qm), cmp)
    heads = [R.check_out(g.double(), torch.from_numpy(r).double(), b, f"head {j}")
             for j, (g, r, b) in enumerate(zip(fms, ref, cmp.pop("head_bounds")))]
    e4 = [v for v in cmp.values() if "exact_checked" in v]
    summary = {"min_exact_checked": min(v["exact_checked"] for v in e4), "worst_ulps": max(v["worst_ulps"] for v in e4),
               "near_zero_beyond_one_ulp": sum(v["near_zero_beyond_one_ulp"] for v in e4),
               "fp16_worst_err_over_bound": max(v["worst_err_over_bound"] for v in cmp.values() if "worst_err_over_bound" in v),
               "heads_worst_err_over_bound": max(heads)}
    _record(f"fp8_layers_416_{weights}", {"layers": {str(k): v for k, v in cmp.items()}, "summary": summary})
    print(f"FP8LAYERS {weights}: {summary}")


# End-to-end bars, about 2x the values measured on an H100 80GB HBM3 (700 W), 416 x 416, batch 2: max-norm of the
# logits per feature map, and the 99.9th percentile of the element-wise errors of boxes (16 px floor), confidences and
# probabilities (1e-2 floor); the maxima are recorded.  Without teacher forcing, the oracle and the engine drift apart:
# where the two accumulation orders put a value on different sides of an e4m3 rounding midpoint, the outputs differ by
# one ulp (6-12 %), and such flips propagate through the 70 e4m3 layers.  test_network_layers_vs_fake_quant_oracle is
# the per-layer check; this one bounds the drift.  cfg2 (heads x8, random BN) amplifies logit differences in exp / sigmoid.
_FQ_BARS = {"cfg1": (0.36, 0.32, 0.06, 0.06), "cfg2": (0.40, 30.0, 3.4, 38.0)}
# The fp8 engine against the fp16 engine: the quantization error itself with random weights (measured 0.11-0.21
# max-norm), reported, with a generous bar.
_FP16_BARS = {"cfg1": 0.5, "cfg2": 0.5}


@pytest.mark.parametrize("weights", ["cfg1", "cfg2"])
def test_network_parity_416(weights):
    x, m, qm = _cached_models(weights)
    xt = torch.from_numpy(x).cuda()
    got = [f.cpu().numpy() for f in qm.forward(xt)]
    act, wts = qm.fp8_scales()["act"], qm.fp8_scales()["weight"]
    ref = fq_forward(x, _params(weights), [a[2] for a in act], wts)
    fp16 = [f.cpu().numpy() for f in m.forward(xt)]
    rec = {"vs_fake_quant_oracle": _compare(got, ref, 416), "vs_fp16_engine": _compare(got, fp16, 416)}
    _record(f"fp8_forward_416_{weights}", rec)
    print(json.dumps(rec))
    mn, bb, bc, bp = _FQ_BARS[weights]
    r = rec["vs_fake_quant_oracle"]
    for k in ("fm1", "fm2", "fm3"):
        assert r[k + "_maxnorm"] < mn, (k, r)
    assert r["boxes"]["p999"] < bb and r["confs"]["p999"] < bc and r["probs"]["p999"] < bp, r
    for k in ("fm1", "fm2", "fm3"):
        assert rec["vs_fp16_engine"][k + "_maxnorm"] < _FP16_BARS[weights]


@pytest.mark.parametrize("cn,n,h,w,thr", [(80, 2, 64, 96, 0.3), (80, 3, 128, 160, 0.3), (80, 2, 416, 416, 0.3),
                                          (80, 1, 96, 64, 0.05), (20, 2, 96, 96, 0.3), (80, 2, 64, 64, 0.0)])
def test_fp8_detect_fused_equals_unfused(cn, n, h, w, thr):
    """detect_raw on the quantized model is bit-identical to forward -> predict_scores -> batched_nms_raw."""
    from yolov3_tensorflow_b200.utils.nms_utils import batched_nms_raw
    x = torch.from_numpy(gen_inputs(5 + h, n, h, w)).cuda()
    _, qm = _models("cfg2", [gen_inputs(77, 2, h, w)], cn)
    mb = 20
    boxes, scores = qm.predict_scores(qm.forward(x))
    ub = batched_nms_raw(boxes, scores, cn, mb, thr, 0.45)
    fb = qm.detect_raw(x, mb, thr, 0.45)
    assert torch.equal(fb[0], boxes)
    cu, cf = ub[4].cpu().numpy(), fb[5].cpu().numpy()
    assert np.array_equal(cu, cf), (cu, cf)
    for i in range(n):
        k = int(cu[i])
        for a, b in zip(ub[:4], fb[1:5]):
            assert torch.equal(a[i, :k], b[i, :k])
    dets = qm.detect(x, mb, thr, 0.45)
    assert len(dets) == n


def test_fp8_detect_graphed_equals_eager():
    _, qm = _models("cfg2", [gen_inputs(3, 2, 96, 128)])
    for seed in (1, 2):
        x = torch.from_numpy(gen_inputs(seed, 1, 96, 128)).cuda()
        e = [t.clone() for t in qm.detect_raw(x, 20, 0.3, 0.45)]
        g = qm.detect_graphed(x, 20, 0.3, 0.45)
        for a, b in zip(e, g):
            assert torch.equal(a, b)


# ------------------------------------------------------------------------- API
def test_fp8_api():
    """Training and parameter changes on the quantized model raise ValueError; calibrating at 416 and running at 608
    works; the source model's fp16 detections are unchanged by quantize_fp8."""
    import yolov3_tensorflow_b200 as pkg
    m = pkg.yolov3(80, O.COCO_ANCHORS, dtype="fp16")
    m.set_params(_params("cfg2"), "HWIO")
    x416 = torch.from_numpy(gen_inputs(9, 1, 416, 416)).cuda()
    before = [t.clone() for t in m.detect_raw(x416)]
    qm = m.quantize_fp8(x416)
    after = m.detect_raw(x416)
    k = int(before[5][0])
    assert torch.equal(before[0], after[0]) and torch.equal(before[5], after[5]) and k > 0
    for a, b in zip(before[1:5], after[1:5]):
        assert torch.equal(a[0, :k], b[0, :k])
    x608 = torch.from_numpy(gen_inputs(10, 2, 608, 608)).cuda()
    out = qm.detect_raw(x608)
    assert out[0].shape[0] == 2 and int(out[5].sum()) >= 0
    fms = qm.forward(x608)
    assert all(bool(torch.isfinite(f).all()) for f in fms)
    ys = [torch.zeros(1, 416 // s, 416 // s, 3, 86, device="cuda") for s in (32, 16, 8)]
    with pytest.raises(ValueError, match="quantize"):
        qm.forward(x416, is_training=True)
    with pytest.raises(ValueError, match="quantize"):
        qm.train_step(x416, ys, 1e-3)
    with pytest.raises(ValueError, match="quantize"):
        next(qm.train_step_sync_bn(x416, ys, 1e-3, 1))
    with pytest.raises(ValueError, match="quantize"):
        qm.set_params(_params("cfg2"), "HWIO")
    with pytest.raises(ValueError, match="quantize"):
        qm.init_params(0)
    with pytest.raises(ValueError, match="quantize"):
        pkg.load_weights(qm, "/nonexistent.weights")
    with pytest.raises(ValueError):
        pkg.yolov3(80, O.COCO_ANCHORS, dtype="e4m3")


def test_fp8_plan_without_scales_fails(L):
    """A bound e4m3 plan whose activation scales were never set refuses to run."""
    h = C.c_void_p()
    L.check(L.lib.yb_net_create(C.byref(h), 80, 1, 64, 64, L.YB_E4M3, 0), "create")
    try:
        a, p = C.c_size_t(), C.c_size_t()
        L.check(L.lib.yb_net_arena_bytes(h, C.byref(a), C.byref(p)), "arena")
        act = torch.zeros(a.value, dtype=torch.uint8, device="cuda")
        par = torch.zeros(p.value, dtype=torch.uint8, device="cuda")
        L.check(L.lib.yb_net_bind(h, L.ptr(act), a.value, L.ptr(par), p.value, None), "bind")
        x = torch.zeros(1, 64, 64, 3, device="cuda")
        fm = [torch.empty(1, 64 // s, 64 // s, 255, device="cuda") for s in (32, 16, 8)]
        rc = L.lib.yb_net_forward(h, L.ptr(x), L.ptr(fm[0]), L.ptr(fm[1]), L.ptr(fm[2]), None)
        assert rc == -1 and b"scales" in L.lib.yb_last_error_string()
    finally:
        L.lib.yb_net_destroy(h)
